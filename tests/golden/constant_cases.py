"""Input frames of the constant-advection golden cases (gen_constant_golden.py), shared by the
generator and the tests.  Every case is rebuilt from its seed and generator arguments."""
import numpy as np

from pysteps_b200 import _synthetic as syn

CASES = [
    "shift_256_f64", "shift_256_f32", "shift_1024_f64", "shift_1024_f32", "shift_2048_f64", "shift_2048_f32",
    "three_frames_192x160", "nan_blocks_edges_200x180", "masked_128x96", "all_nan_32x32",
    "constant_inexact_mean_37x41", "single_finite_24x20", "one_by_one", "one_row_1x57", "one_column_43x1",
    "odd_width_31x97", "rotation_160x160",
]

# the cases whose frames have more than 2^20 pixels (slow on the CPU oracle)
LARGE = ("shift_2048_f64", "shift_2048_f32")

# Cases whose Nelder-Mead path is decided by the summation order of the centred sums, which the
# reference leaves to BLAS: two evaluations (indices into the recorded sequence) at different points
# where the true correlation is exactly 1 -- the overlaps differ only by a border row or column of a
# perfect shift -- so f = -1 up to one ulp; the reference and the fixed device order round the two
# differently and Nelder-Mead goes on from a different vertex.  Both paths end on the plateau f = -1.
ORDER_DECIDED = {
    "shift_1024_f64": (13, 16),   # v = (-2.625, 1.625) and (-2.53125, 2.15625)
    "shift_1024_f32": (13, 16),
    "masked_128x96": (13, 15),    # v = (-1.25, 3.125) and (-1.25, 2.625)
    "odd_width_31x97": (6, 7),    # v = (1, -1) and (0.5, -1.5)
}


def _rotated(r, angle):
    """r sampled at the pixel grid rotated by `angle` about the centre (nearest pixel, zero outside)."""
    m, n = r.shape
    y, x = np.mgrid[0:m, 0:n].astype(np.float64)
    yc, xc = (m - 1) / 2.0, (n - 1) / 2.0
    c, s = np.cos(angle), np.sin(angle)
    ys = np.rint(yc + c * (y - yc) - s * (x - xc)).astype(np.int64)
    xs = np.rint(xc + s * (y - yc) + c * (x - xc)).astype(np.int64)
    ok = (ys >= 0) & (ys < m) & (xs >= 0) & (xs < n)
    out = np.zeros_like(r)
    out[ok] = r[ys[ok], xs[ok]]
    return out


def build_case(name):
    """-> R, the (T, m, n) input of constant()"""
    if name.startswith("shift_"):
        _, size, dt = name.split("_")
        size = int(size)
        R = syn.rain_frames(size, size, 2, seed=size, dx=3, dy=-2)
        return R.astype(np.float32) if dt == "f32" else R
    if name == "three_frames_192x160":
        return syn.rain_frames(192, 160, 3, seed=5, dx=-2, dy=1)
    if name == "nan_blocks_edges_200x180":
        R = syn.rain_frames(200, 180, 2, seed=6, dx=2, dy=2)
        R[0, 40:70, 100:150] = np.nan
        R[1, 120:160, 20:60] = np.nan
        R[1, :, :3] = np.nan
        R[0, -2:, :] = np.nan
        R[1, 0, :] = np.nan
        return R
    if name == "masked_128x96":
        R = syn.rain_frames(128, 96, 2, seed=7, dx=1, dy=-3)
        R[1, 10:20, 10:30] = np.nan
        mask = np.zeros(R.shape, bool)
        mask[1, 5:25, 5:40] = True     # over NaN and finite values of the last frame
        mask[0, 60:90, 50:80] = True   # over finite values of the frame that is shifted
        mask[1, 100:110, :] = True
        return np.ma.MaskedArray(R, mask=mask)
    if name == "all_nan_32x32":
        R = syn.rain_frames(32, 32, 2, seed=8)
        R[1] = np.nan
        return R
    if name == "constant_inexact_mean_37x41":
        return np.full((2, 37, 41), 0.1)
    if name == "single_finite_24x20":
        R = np.full((2, 24, 20), np.nan)
        R[:, 11, 7] = 2.5
        return R
    if name == "one_by_one":
        return np.array([[[1.5]], [[2.0]]])
    if name == "one_row_1x57":
        return syn.rain_frames(1, 57, 2, seed=9, dx=2, dy=0) + np.arange(57)
    if name == "one_column_43x1":
        return syn.rain_frames(43, 1, 2, seed=10, dx=0, dy=1) + np.arange(43)[:, None]
    if name == "odd_width_31x97":
        return syn.rain_frames(31, 97, 2, seed=11, dx=-1, dy=1)
    if name == "rotation_160x160":
        r0 = syn.rain_field(160, 160, 12)
        return np.stack([r0, _rotated(r0, 0.05)])
    raise KeyError(name)
