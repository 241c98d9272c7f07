"""GPU tests of the corner selection kernel (b200_good_features, csrc/lk_features.cu) by itself, on
synthetic float32 minimum-eigenvalue maps, against the oracle's cv2.goodFeaturesToTrack restatement
(oracle/lucaskanade.py, pinned to the cv2 binary in tests/test_oracle_lk.py).  Bar: the same corner
count and the corners bit for bit, in order.

The parameters choose the code that runs, and every choice is exercised here:
  smem    select_smem_kernel: min_distance >= 1, round(min_distance) <= 32, cell grid <= 200 KB
  global  select_kernel with the grid in global memory: a larger grid or cell
  nodist  select_kernel without a distance test: min_distance < 1
and the bitonic sort's global passes (more than 2048 candidates)."""
import math

import numpy as np
import pytest
from conftest import assert_bits_equal

pytestmark = pytest.mark.gpu

SMEM_GRID_BYTES = 200 * 1024


def _path(m, n, md):
    """The kernel b200_good_features picks for an m x n map (the host's own rule)."""
    if not md >= 1.0:
        return "nodist"
    cell = round(md)  # cvRound: half to even, like lrint
    ncell = ((n + cell - 1) // cell) * ((m + cell - 1) // cell)
    return "smem" if cell <= 32 and ncell * 4 <= SMEM_GRID_BYTES else "global"


def _ncand(eig, valid, quality):
    """Number of candidates (thresholded 3x3 local maxima inside the mask, off the border)."""
    from oracle import lucaskanade as ora
    return len(ora.good_features_to_track(None, valid, 0, quality, 0.0, eig=eig))


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _lib


def _select(env, eig, valid, maxc, quality, md):
    torch, L = env
    m, n = eig.shape
    de = torch.from_numpy(np.ascontiguousarray(eig, np.float32)).cuda()
    dv = None if valid is None else torch.from_numpy(np.ascontiguousarray(valid, np.uint8)).cuda()
    out = torch.full((maxc, 2), -1.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    L.call("b200_good_features", de.data_ptr(), None if dv is None else dv.data_ptr(), m, n, maxc,
           float(quality), float(md), out.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream().cuda_stream)
    c = int(cnt.item())
    assert 0 <= c <= maxc, c
    return out[:c].cpu().numpy()


def _check(env, eig, valid, maxc, quality, md, what=""):
    from oracle import lucaskanade as ora
    got = _select(env, eig, valid, maxc, quality, md)
    want = ora.good_features_to_track(None, valid, maxc, quality, md, eig=eig)
    tag = f"{what} {eig.shape} maxc={maxc} quality={quality} md={md!r} path={_path(*eig.shape, md)}"
    assert len(got) == len(want), f"{tag}: corner count {len(got)} != {len(want)}"
    assert_bits_equal(got, want, tag)
    return want


def _noise_map(m, n, seed, levels=None):
    """Every pixel random: about one pixel in nine is a candidate, at every distance from the others.
    With `levels`, values are drawn from that many levels: plateaus and ties everywhere."""
    rng = np.random.default_rng(seed)
    if levels:
        return (rng.integers(1, levels + 1, (m, n)) / levels).astype(np.float32)
    return rng.random((m, n), dtype=np.float32) + np.float32(1e-3)


def _lattice_map(m, n, count, seed, equal=False, spacing=2):
    """`count` isolated peaks (distinct values unless `equal`) on a lattice, zero elsewhere."""
    ys, xs = np.mgrid[1:m - 1:spacing, 1:n - 1:spacing]
    pos = np.stack([ys.ravel(), xs.ravel()], 1)
    assert count <= len(pos), (count, len(pos))
    rng = np.random.default_rng(seed)
    pos = pos[rng.permutation(len(pos))[:count]]
    eig = np.zeros((m, n), np.float32)
    vals = np.ones(count) if equal else (1.0 + rng.permutation(count)) / count
    eig[pos[:, 0], pos[:, 1]] = vals.astype(np.float32)
    return eig


# ---------------------------------------------------------------------------------- every path
@pytest.mark.parametrize("shape,md,path", [
    ((256, 256), 10.0, "smem"),
    ((256, 256), 4.5, "smem"),
    ((1024, 1024), 4.0, "global"),   # 65 536 cells = 256 KB
    ((256, 256), 33.0, "global"),    # cell > 32
    ((256, 256), 40.5, "global"),
    ((256, 256), 0.0, "nodist"),
    ((256, 256), 0.5, "nodist"),
    ((256, 256), 0.99999999999, "nodist"),
    ((200, 200), 1.0, "smem"),
    ((256, 256), 1.0, "global"),     # 1-px cells: 65 536 of them
])
@pytest.mark.parametrize("levels", [None, 3])
def test_each_selection_path(env, shape, md, path, levels):
    assert _path(*shape, md) == path
    eig = _noise_map(*shape, 1, levels)
    assert _ncand(eig, None, 0.01) > 2048  # the bitonic sort's global passes run too
    for maxc in (1000, 5000):
        _check(env, eig, None, maxc, 0.01, md)


# ------------------------------------------------------------------ min_distance whose square is not a float
def _sum_of_two_squares(k):
    for dx in range(int(math.isqrt(k)) + 1):
        dy = math.isqrt(k - dx * dx)
        if dy * dy == k - dx * dx:
            return dx, dy
    return None


def _non_float_min_distances():
    out = []
    for k in (2, 5, 50, 125):
        md = math.sqrt(k)
        out += [md, float(np.nextafter(md, 0.0)), float(np.nextafter(md, 100.0))]
    return out + [10.0 / 3.0]


def _pair_map(m, n, offset, across_batches):
    """Peaks A and B `offset` = (dx, dy) apart, dx, dy >= 0: both survive the greedy selection iff
    their squared distance reaches min_distance^2.  With `across_batches`, 40 isolated filler peaks
    fall between them in the candidate order, so the second of the pair is tested against the grid,
    not inside its batch of 32.
    Far apart: A = 1, B = 0.5, fillers valued between them, far from both.
    Adjacent (|dx|, |dy| <= 1): A and B equal, so that both are 3x3 maxima; B comes first (larger
    raster address), and the fillers, equal too, sit on B's row left of A's column: between them."""
    eig = np.zeros((m, n), np.float32)
    adjacent = max(offset) <= 1
    ax, ay = (n - 4, 40) if adjacent else (40, 40)
    bx, by = ax + offset[0], ay + offset[1]
    eig[ay, ax] = 1.0
    eig[by, bx] = 1.0 if adjacent else 0.5
    if across_batches:
        if adjacent:
            xs = np.arange(1, 1 + 3 * 40, 3)
            assert xs[-1] <= ax - 3
            eig[ay + 1, xs] = 1.0
        else:
            k = 0
            for y in range(100, m - 1, 24):
                for x in range(4, n - 1, 24):
                    if k < 40:
                        eig[y, x] = np.float32(0.6 + 0.3 * k / 40)
                        k += 1
            assert k == 40
    return eig, {(float(ax), float(ay)), (float(bx), float(by))}


@pytest.mark.parametrize("md", _non_float_min_distances())
@pytest.mark.parametrize("path", ["smem", "global"])
@pytest.mark.parametrize("across_batches", [False, True])
def test_non_float_min_distance(env, md, path, across_batches):
    """Peaks exactly floor(md^2) and ceil(md^2) apart.  cv2 compares the squared distance with
    md * md in double; a float threshold accepts or rejects the wrong one."""
    md2 = md * md
    cell = round(md)
    side = 200 if path == "smem" else cell * 230
    assert _path(side, side, md) == path
    # floor(md^2) and ceil(md^2) where they are sums of two squares, and the nearest such
    # squared distances below and at-or-above md^2
    sums = [k for k in range(1, 200) if _sum_of_two_squares(k)]
    ks = {k for k in (math.floor(md2), math.ceil(md2)) if _sum_of_two_squares(k)}
    ks |= {max(k for k in sums if k < md2), min(k for k in sums if k >= md2)}
    for k in sorted(ks):
        eig, pair = _pair_map(side, side, _sum_of_two_squares(k), across_batches)
        want = _check(env, eig, None, 100, 0.01, md, f"d2={k} across_batches={across_batches}")
        kept = pair & {(float(x), float(y)) for x, y in want}
        assert len(kept) == (2 if k >= md2 else 1), (k, md2, want)  # d^2 >= md^2 in double


# ----------------------------------------------------------------------------------------- sort sizes
@pytest.mark.parametrize("count", [1, 2, 2047, 2048, 2049, 4096, 4097, 70000])
def test_sort_sizes(env, count):
    """Isolated peaks with distinct values: the whole candidate order (min_distance 0, every
    candidate kept) and a selection on top of it, across the bitonic local/global pass boundary."""
    m = n = 600 if count > 4097 else 200
    eig = _lattice_map(m, n, count, count)
    assert _ncand(eig, None, 1e-9) == count
    _check(env, eig, None, count, 1e-9, 0.0, "full order")
    _check(env, eig, None, min(count, 3000), 1e-9, 3.0, "smem")
    _check(env, eig, None, min(count, 3000), 1e-9, 33.0, "global")


# ------------------------------------------------------------------------------------------------ ties
@pytest.mark.parametrize("md", [0.0, 2.5, 3.0, 7.0, 33.0])
def test_plateaus_and_equal_peaks(env, md):
    """Plateaus of equal values (every pixel of a plateau that equals its 3x3 dilation is a candidate;
    ties go to the larger raster address first) and equal isolated peaks spread over many batches."""
    for levels in (2, 4):
        _check(env, _noise_map(200, 232, levels, levels), None, 4000, 0.01, md, f"levels={levels}")
    flat = np.zeros((120, 136), np.float32)
    flat[10:60, 20:90] = 0.5
    flat[70:100, 30:40] = 0.5
    _check(env, flat, None, 4000, 0.01, md, "plateau blocks")
    for spacing in (2, 3, 5):
        eig = _lattice_map(160, 200, 1500 if spacing < 5 else 1000, spacing, equal=True, spacing=spacing)
        _check(env, eig, None, 2000, 0.01, md, f"equal peaks spacing {spacing}")


# --------------------------------------------------------------------------------------- max_corners
@pytest.mark.parametrize("shape,md", [((256, 256), 4.0), ((1024, 1024), 4.0), ((256, 256), 0.0)])
def test_max_corners(env, shape, md):
    eig = _noise_map(*shape, 7)
    for maxc in (1, 2, 31, 32, 33, 45, 63, 64, 65, 1000):
        _check(env, eig, None, maxc, 0.01, md)


# ------------------------------------------------------------------ quality, mask and degenerate maps
@pytest.mark.parametrize("md", [0.0, 4.0, 33.0])
def test_quality_mask_and_degenerate_maps(env, md):
    eig = _noise_map(180, 210, 3)
    for quality in (0.0, 1.0, 0.999, 0.5):
        _check(env, eig, None, 3000, quality, md, "quality")
    rng = np.random.default_rng(5)
    masks = {"all": np.ones(eig.shape, np.uint8), "empty": np.zeros(eig.shape, np.uint8),
             "sparse": (rng.random(eig.shape) > 0.3).astype(np.uint8)}
    top = np.unravel_index(np.argmax(eig), eig.shape)
    masks["without the maximum"] = masks["all"].copy()
    masks["without the maximum"][top] = 0
    for name, valid in masks.items():
        _check(env, eig, valid, 3000, 0.01, md, f"mask {name}")
    assert len(_select(env, eig, masks["empty"], 10, 0.01, md)) == 0
    _check(env, np.zeros((64, 80), np.float32), None, 10, 0.01, md, "all-zero map")


@pytest.mark.parametrize("md", [0.0, 4.0, 33.0])
def test_negative_eigenvalue_maps(env, md):
    """cv2's cornerMinEigenVal returns tiny negative values (like -1.5e-8) on straight edges.  With
    the masked maximum negative and quality <= 1 nothing passes the threshold; a quality above 1 puts
    the threshold below the maximum, and the candidates are negative: they must still be ordered by
    value, largest (closest to zero) first."""
    rng = np.random.default_rng(9)
    eig = (-1.5e-8 * (1.0 + 0.2 * rng.random((150, 170)))).astype(np.float32)
    for quality in (0.01, 1.0):
        assert len(_select(env, eig, None, 100, quality, md)) == 0
        _check(env, eig, None, 100, quality, md, "negative, no candidate")
    for quality in (1.5, 2.0):
        assert _ncand(eig, None, quality) > 100
        _check(env, eig, None, 3000, quality, md, "negative candidates")
    # a masked maximum that is negative while the map's maximum outside the mask is positive
    mixed = eig.copy()
    valid = np.ones(eig.shape, np.uint8)
    mixed[50:60, 50:60] = 1.0
    valid[45:65, 45:65] = 0
    _check(env, mixed, valid, 3000, 2.0, md, "negative masked maximum")


# --------------------------------------------------------------------------------------------- shapes
@pytest.mark.parametrize("shape", [(3, 3), (2, 2), (1, 1), (1, 57), (57, 1), (2, 40), (3, 40), (9, 33),
                                   (37, 45), (41, 31), (8, 32), (200, 33)])
@pytest.mark.parametrize("md", [0.0, 1.5, 10.0, 33.0])
def test_shapes(env, shape, md):
    """3x3 has one interior pixel, 2xN and 1xN none; the other sizes are not multiples of the 32x8
    candidate tile."""
    eig = _noise_map(*shape, shape[0] * 1000 + shape[1])
    want = _check(env, eig, None, 50, 0.01, md)
    if min(shape) < 3:
        assert len(want) == 0
    if shape == (3, 3):
        peak = np.zeros((3, 3), np.float32)
        peak[1, 1] = 1.0
        assert len(_check(env, peak, None, 5, 0.01, md, "single interior peak")) == 1


# ------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("md", [math.sqrt(50), 0.5, math.sqrt(5)])
def test_detection_and_sparse_lk_with_min_distance(env, md):
    from oracle import lucaskanade as ora
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200 import stages
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    for seed, (m, n) in enumerate([(200, 224), (257, 300)]):
        fr = syn.rain_frames(m, n, 2, 40 + seed, dx=2, dy=-1)
        a = np.ma.masked_invalid(fr[0])
        np.ma.set_fill_value(a, a.min())
        got = stages.detection(a, min_distance=md)
        want = ora.detection(a, min_distance=md)
        assert len(got) == len(want) and len(want) > 0
        assert_bits_equal(np.asarray(got, np.float32), want, f"detection md={md!r}")
        kw = dict(dense=False, fd_kwargs={"min_distance": md})
        xy, uv = lk(fr, **kw)
        with ora.knn_mode("ckdtree"):
            oxy, ouv = ora.dense_lucaskanade(fr, **kw)
        assert np.array_equal(xy, oxy) and np.array_equal(uv, ouv), (m, n, md)
