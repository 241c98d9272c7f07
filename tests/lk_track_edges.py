"""The edge grid of the pyramidal Lucas-Kanade tracker (csrc/lk_track.cu, a restatement of
cv::calcOpticalFlowPyrLK): frames, points and parameters at which the kernel changes branch.

  windows   nchunk = ww / 8 == 0 (3x3, 7x7, 4x40), ntail = ww % 8 == 0 (8, 16, 64 wide), the largest
            shared-memory footprints (64x64, 63x65, 3x1365), div_small divisors beyond 64 (100, 1365)
  levels    0, 1, 3, 5, more than the geometry allows, and 8 / 10 at 1024^2 with a 3x3 window
            (nine levels: deeper than the eight the level arrays once held)
  criteria  COUNT and/or EPS, max_count 0, 1, 100 and clamped from 500 and -5, epsilon clamped
            from 20; min_eig_thr 0 .. 1e-2
  frames    smaller than the window, odd sizes, flat (status 0 through D / minEig), saturated
  points    corners, window origins at -ww, -ww-1, w-1 and w on both axes at level 0 and at the
            coarsest level, NaN, +-inf, +-3e9, -0.0

tests/test_oracle_lk_track_edges.py pins the oracle to live cv2 on this grid (CPU);
tests/test_lk_track_edges_gpu.py holds the device to the oracle on it.  Nothing here imports cv2:
the GPU machines do not have it."""
import functools

import numpy as np

from oracle import lucaskanade as ora
from pysteps_b200 import _synthetic as syn


def pyramid_sizes(m, n, win, nr_levels):
    """[(h, w)] of the levels cv::buildOpticalFlowPyramid keeps: halve while both sides exceed the
    window, at most nr_levels times."""
    sizes = [(m, n)]
    while len(sizes) <= nr_levels:
        h, w = sizes[-1]
        nh, nw = (h + 1) // 2, (w + 1) // 2
        if nw <= win[0] or nh <= win[1]:
            break
        sizes.append((nh, nw))
    return sizes


def _textured(m, n, seed):
    """uint8 power-law texture I and J = I resampled (bilinear, float64) under a sub-pixel,
    spatially varying shift, plus integer noise."""
    rng = np.random.default_rng(seed)
    base = syn.powerlaw_field(m, n, seed)
    I = np.clip((base - base.min()) / (base.max() - base.min()) * 255, 0, 255).astype(np.uint8)
    yy, xx = np.mgrid[0:m, 0:n].astype(np.float64)
    mx = np.clip(xx - 2.37 + 0.8 * np.sin(yy / 40.0), 0, n - 1.001)
    my = np.clip(yy + 1.61 + 0.6 * np.cos(xx / 55.0), 0, m - 1.001)
    x0, y0 = np.floor(mx).astype(int), np.floor(my).astype(int)
    tx, ty = mx - x0, my - y0
    f = I.astype(np.float64)
    x1, y1 = np.minimum(x0 + 1, n - 1), np.minimum(y0 + 1, m - 1)
    J = (f[y0, x0] * (1 - tx) * (1 - ty) + f[y0, x1] * tx * (1 - ty) +
         f[y1, x0] * (1 - tx) * ty + f[y1, x1] * tx * ty)
    J = np.clip(np.rint(J) + rng.integers(-6, 7, J.shape), 0, 255).astype(np.uint8)
    return I, J


def _checker(m, n):
    return ((np.indices((m, n)).sum(0) % 2) * 255).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def frames(name):
    """(I, J) uint8 frame pair by name"""
    if name == "tex300x340":
        return _textured(300, 340, 9)
    if name == "tex1024":
        return _textured(1024, 1024, 3)
    if name == "small20x26":
        return _textured(20, 26, 4)
    if name == "odd37x53":
        return _textured(37, 53, 5)
    if name == "flat64x80":
        z = np.zeros((64, 80), np.uint8)
        return z, z.copy()
    if name == "checker_shift":
        c = _checker(64, 80)
        return c, np.roll(c, 1, 1)
    if name == "checker_inverted":
        c = _checker(64, 80)
        return c, 255 - c
    raise KeyError(name)


SPECIAL = np.array([[np.nan, 10.0], [10.0, np.nan], [np.nan, np.nan], [np.inf, 5.0], [-np.inf, 5.0],
                    [5.0, np.inf], [5.0, -np.inf], [3e9, 4.0], [-3e9, 4.0], [4.0, 3e9], [4.0, -3e9],
                    [-0.0, -0.0], [-0.0, 7.5], [12.25, -0.0]], np.float32)


def boundary_points(m, n, win, nr_levels):
    """Points whose window origin floor(x / 2^L - (ww - 1) / 2) is -ww, -ww-1, w_L-1 and w_L (and
    the same in y) at level 0 and at the coarsest level L, exactly on and half a pixel past the
    integer; the other coordinate sits mid-frame."""
    sizes = pyramid_sizes(m, n, win, nr_levels)
    half = ((win[0] - 1) * 0.5, (win[1] - 1) * 0.5)
    out = []
    for level in sorted({0, len(sizes) - 1}):
        h, w = sizes[level]
        s = float(1 << level)
        for axis, (ext, wsz) in enumerate(((w, win[0]), (h, win[1]))):
            for target in (-wsz, -wsz - 1, ext - 1, ext):
                for frac in (0.0, 0.5):
                    p = [n * 0.5, m * 0.5]
                    p[axis] = (target + frac + half[axis]) * s
                    out.append(p)
    return np.array(out, np.float32)


def points(name, I, win, nr_levels, max_corners=300):
    """detected corners + window-origin boundary points + NaN / inf / huge / -0.0 points"""
    m, n = I.shape
    parts = [ora.good_features_to_track(I, None, max_corners, 0.01, 7), boundary_points(m, n, win, nr_levels)]
    if name.startswith("small"):
        parts.append(np.array([[0, 0], [n - 1, m - 1], [-3, 4], [n + 4, 10]], np.float32))
    parts.append(SPECIAL)  # last: tests find them there
    return np.ascontiguousarray(np.concatenate(parts).astype(np.float32))


def _case(frame, win, levels, criteria=(3, 10, 0), min_eig=1e-4, max_corners=300):
    tag = f"{frame}-w{win[0]}x{win[1]}-L{levels}-c{criteria[0]}_{criteria[1]}_{criteria[2]}-e{min_eig:g}"
    return tag, dict(frame=frame, win=win, levels=levels, criteria=criteria, min_eig=min_eig,
                     max_corners=max_corners)


CASES = dict([
    # windows: nchunk 0, ntail 0, the largest shared-memory footprints, divisors 100 and 1365
    *[_case("tex300x340", win, 2) for win in ((3, 3), (7, 7), (8, 8), (16, 16), (64, 64), (64, 8), (8, 64),
                                               (4, 40), (40, 4), (100, 30), (1365, 3), (3, 1365), (63, 65))],
    # levels, and more levels than the geometry allows (a 7x7 window stops 300x340 at level 5)
    *[_case("tex300x340", (7, 7), lv) for lv in (0, 1, 3, 5, 9)],
    # nine levels at 1024^2 with a 3x3 window: level 7 alone tracks a different set of points
    *[_case("tex1024", (3, 3), lv, max_corners=100) for lv in (7, 8, 10)],
    # criteria: COUNT / EPS alone, max_count 0, 1, 100 and clamped, epsilon above 10
    *[_case("tex300x340", (21, 21), 3, crit) for crit in ((3, 10, 0.03), (1, 10, 0), (2, 10, 0.01), (3, 0, 0),
                                                          (3, 1, 0), (3, 100, 0), (3, 500, 0), (1, -5, 0),
                                                          (3, 10, 20.0))],
    *[_case("tex300x340", (21, 21), 3, min_eig=me) for me in (0.0, 1e-3, 1e-2)],
    # frames smaller than the window, odd sizes, flat and saturated frames
    *[_case("small20x26", win, 3) for win in ((21, 21), (25, 17), (3, 3))],
    _case("odd37x53", (5, 5), 4),
    _case("flat64x80", (21, 21), 2),
    _case("checker_shift", (21, 21), 2),
    _case("checker_inverted", (8, 8), 1, (3, 10, 0.01)),
])


def case_inputs(tag):
    """(I, J, points, case dict) of a grid case"""
    c = CASES[tag]
    I, J = frames(c["frame"])
    return I, J, points(c["frame"], I, c["win"], c["levels"], c["max_corners"]), c
