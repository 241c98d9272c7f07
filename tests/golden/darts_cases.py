"""Input frames and keyword arguments of the DARTS golden cases (gen_darts_golden.py), shared by the
generator and the tests.  Every case is rebuilt from its seed and generator arguments."""
import numpy as np

from pysteps_b200 import _synthetic as syn

CASES = [
    "shift_256_f64", "shift_256_f32", "shift_2048_f64", "t9_nt6_192x160", "alias_80x90", "odd_97x131",
    "small_64x48", "lsq1_128x128", "spectral_128x112", "rotation_160x160", "all_equal_96x96", "masked_nan_128x96",
    "m5_256x224", "fx_tiles_160x256", "t2_nt0_96x80", "alias_fill_12x9",
]

# The golden keeps the file small without losing the field: the reference's field is
# real(numpy.fft.ifft2(_fill(.))) of its solution x, so it stores x and the generator asserts that
# reference_field(x) rebuilds the reference's result bit for bit.  It also stores the field itself at
# seeded pixels (4096 above 2^20 pixels, else 256) as a check of the rebuild, and MM by its upper
# triangle (MM is Hermitian).
# the cases whose reference run raises (the golden stores the exception)
RAISES = ("masked_nan_128x96",)


def _rotating(m, n, T, seed, step):
    r0 = syn.rain_field(m, n, seed)
    y, x = np.mgrid[0:m, 0:n].astype(np.float64)
    yc, xc = (m - 1) / 2.0, (n - 1) / 2.0
    out = []
    for t in range(T):
        c, s = np.cos(step * t), np.sin(step * t)
        ys = np.rint(yc + c * (y - yc) - s * (x - xc)).astype(np.int64)
        xs = np.rint(xc + s * (y - yc) + c * (x - xc)).astype(np.int64)
        ok = (ys >= 0) & (ys < m) & (xs >= 0) & (xs < n)
        f = np.zeros_like(r0)
        f[ok] = r0[ys[ok], xs[ok]]
        out.append(f)
    return np.stack(out)


def build_case(name):
    """-> (R, kwargs): the (T, m, n) input of DARTS and its keyword arguments (verbose=False added)"""
    kw = {"verbose": False}
    if name.startswith("shift_"):
        _, size, dt = name.split("_")
        size = int(size)
        R = syn.rain_frames(size, size, 6, seed=size + 1, dx=3, dy=-2)
        return (R.astype(np.float32) if dt == "f32" else R), kw
    if name == "t9_nt6_192x160":
        return syn.rain_frames(192, 160, 9, seed=21, dx=-2, dy=1), dict(kw, N_t=6)
    if name == "alias_80x90":
        return syn.rain_frames(80, 90, 6, seed=22, dx=1, dy=2), kw
    if name == "odd_97x131":
        return syn.rain_frames(97, 131, 6, seed=23, dx=-1, dy=-1), kw
    if name == "small_64x48":
        return syn.rain_frames(64, 48, 6, seed=24, dx=2, dy=0), dict(kw, N_x=10, N_y=10, M_x=1, M_y=2)
    if name == "lsq1_128x128":
        return syn.rain_frames(128, 128, 6, seed=25, dx=2, dy=-1), dict(kw, lsq_method=1)
    if name == "spectral_128x112":
        return syn.rain_frames(128, 112, 6, seed=26, dx=-3, dy=1), dict(kw, output_type="spectral")
    if name == "rotation_160x160":
        return _rotating(160, 160, 6, 27, 0.03), kw
    if name == "all_equal_96x96":
        return np.full((6, 96, 96), 0.3), kw
    if name == "masked_nan_128x96":
        R = syn.rain_frames(128, 96, 6, seed=28, dx=1, dy=-3)
        R[2, 10:20, 10:30] = np.nan
        mask = np.zeros(R.shape, bool)
        mask[2, 5:25, 5:40] = True
        return np.ma.MaskedArray(R, mask=mask), kw
    if name == "m5_256x224":  # the most unknowns supported: n_c = 242
        return syn.rain_frames(256, 224, 6, seed=29, dx=2, dy=1), dict(kw, N_x=30, N_y=30, M_x=5, M_y=5)
    if name == "fx_tiles_160x256":  # fx = 73: a second 64-wide frequency tile of the x pass
        return syn.rain_frames(160, 256, 6, seed=30, dx=-2, dy=2), dict(kw, N_x=70, M_x=2, N_y=20)
    if name == "t2_nt0_96x80":  # T = 2 admits only N_t = 0; y = k_t X is then zero, so is the field: MM holds
        return syn.rain_frames(96, 80, 2, seed=31, dx=1, dy=1), dict(kw, N_t=0)
    if name == "alias_fill_12x9":  # M_x = 5 on n = 9: _fill puts several coefficients on one column
        return syn.rain_frames(12, 9, 4, seed=32, dx=1, dy=0), dict(kw, N_t=1, N_x=2, N_y=3, M_x=5, M_y=2)
    raise KeyError(name)


def sample_pixels(m, n, seed=2048):
    """(ys, xs) of the seeded pixels at which the golden stores the field"""
    count = 4096 if m * n > 1 << 20 else 256
    rng = np.random.default_rng(seed)
    return rng.integers(0, m, count), rng.integers(0, n, count)


def reference_field(x, kw, m, n):
    """What the reference returns for its solution x (darts.py:197-220) with numpy's FFT: the
    (2, h, w) coefficients for output_type="spectral", else real(ifft2(_fill(.))) of U and V."""
    M_x, M_y = kw.get("M_x", 2), kw.get("M_y", 2)
    h, w = 2 * M_y + 1, 2 * M_x + 1
    V, U = x[: h * w].reshape(h, w), x[h * w: 2 * h * w].reshape(h, w)
    if kw.get("output_type", "spatial") == "spectral":
        return np.stack([U, V])
    k_x, k_y = np.meshgrid(np.arange(-M_x, M_x + 1), np.arange(-M_y, M_y + 1))
    out = []
    for C in (U, V):
        X_f = np.zeros((m, n), dtype=complex)
        X_f[k_y, k_x] = C
        out.append(np.real(np.fft.ifft2(X_f)))
    return np.stack(out)


def hermitian_from_upper(up):
    """the (n, n) Hermitian matrix whose upper triangle, row by row, is up"""
    nc = int(round((np.sqrt(8 * len(up) + 1) - 1) / 2))
    iu = np.triu_indices(nc)
    out = np.zeros((nc, nc), dtype=up.dtype)
    out[iu[1], iu[0]] = np.conj(up)
    out[iu] = up
    return out


def golden_matrix(g, name, key):
    """MM or Mhy of a case"""
    return hermitian_from_upper(g[name + "/MM_upper"]) if key == "MM" else g[name + "/Mhy"]


# Bars, relative to the largest magnitude the golden holds: float64 fields (lsq_method 2) 1e-11;
# lsq_method 1, whose conditioning the Gram matrix squares, 1e-10; float32 frames 1e-6 (the
# reference's FFT runs in complex64 for them).  MM and M^H y: 1e-12 (1e-6 for float32 frames).
def field_bar(name):
    return 1e-6 if name.endswith("_f32") else (1e-10 if name.startswith("lsq1") else 1e-11)


def matrix_bar(name):
    return 1e-6 if name.endswith("_f32") else 1e-12


def field_error(name, got, g, R, kw):
    """(max |got - reference|, max |reference|): the whole field against the reference's, rebuilt from
    its x, and the field at the stored pixels against the reference's values there"""
    got = np.asarray(got)
    m, n = R.shape[1:]
    want = reference_field(g[name + "/x"], kw, m, n)
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, got.dtype, want.shape, want.dtype)
    d = float(np.abs(got - want).max())
    if kw.get("output_type", "spatial") == "spatial":
        ys, xs = sample_pixels(m, n)
        d = max(d, float(np.abs(got[:, ys, xs] - g[name + "/pixels"]).max()))
    return d, float(np.abs(want).max())


def matrix_error(a, want):
    """(max |a - want|, max |want|)"""
    return float(np.abs(np.asarray(a) - want).max()), float(np.abs(want).max())
