"""GPU: the three DARTS entry points (csrc/darts.cu) at the edges of their tiles and parameters,
against the extended-precision references and a-priori bounds of darts_exact.py (their CPU checks are
tests/test_darts_bound.py).  Every output and work buffer starts as NaN, so a tile that is never
written shows.

  spectrum   frequency tiles of darts_rows_kernel across XF = 64 (fx = 64 .. 129), conjugate reads
             with odd and even n, frames narrower than one XK = 16 step, 1-pixel axes, K_t = 2(T-2)+1
             and T = 2, darts_cols_kernel's K_y and K_x either side of 16 and 32, float32 frames,
             a 1e4 offset and an extreme frames[0, 0, 0], and a sampled 2048^2 case with four
             frequency tiles: every entry within its bound
  normal     on those spectra and on random blocks spanning 2^-30 .. 2^30: bit-identical to the
             restatement of darts_normal_kernel, within the bound of the longdouble M^H M and M^H y,
             MM Hermitian bit for bit with a +0.0 imaginary diagonal; M up to 5 (n_c = 242),
             asymmetric M, rows 1, 27, 511, 513, and 66 row blocks
  synthesize 1x1 on 1x1 up to w = 121 (the widest accepted) and n = 1000, within the bound; zero
             coefficients give exact zeros; fill_tables' colliding placement; w = 122 is refused

Largest error / bound seen on an H100 80GB HBM3 (700 W power limit): spectrum 1.6e-2 (m1; 1.4e-4 at
2048^2), normal equations 3.6e-2 (rows511_m55), synthesis 1.1e-1 (1x1 on 1x1).  Each test prints its
ratio (-s)."""
import numpy as np
import pytest

import darts_exact as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _device, _lib


def _up(env, a):
    torch = env[0]
    return torch.from_numpy(np.array(a, order="C")).cuda()  # a copy: the twiddle tables are read-only


def _nan(env, n, dtype):
    torch = env[0]
    return torch.full((n,), complex("nan+nanj") if dtype.is_complex else float("nan"), dtype=dtype,
                      device="cuda")


def _spectrum(env, R, N_x, N_y, N_t, M_x, M_y):
    """b200_darts_spectrum into NaN-filled buffers -> (block, tables)"""
    from pysteps_b200.motion import darts as dm
    torch, dev, L = env
    T, m, n = R.shape
    tw_x, tw_y, tw_t, K = dm.spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y)
    fx, Ky, Kt, Kx = tw_x.shape[0], tw_y.shape[0], tw_t.shape[0], 2 * K + 1
    frames = _up(env, R)
    tabs = [_up(env, t) for t in (tw_x, tw_y, tw_t)]
    work = _nan(env, T * m * fx + Kt * m * Kx, torch.complex128)
    spec = _nan(env, Kt * Ky * Kx, torch.complex128)
    L.call("b200_darts_spectrum", frames.data_ptr(), dev.dtype_code(frames.dtype), T, m, n, tabs[0].data_ptr(), fx,
           tabs[1].data_ptr(), Ky, tabs[2].data_ptr(), Kt, K, work.data_ptr(), spec.data_ptr(), dev.stream_ptr())
    return spec.cpu().numpy().reshape(Kt, Ky, Kx), (tw_x, tw_y, tw_t, K)


def _normal(env, X, N_x, N_y, N_t, M_x, M_y, sx, sy):
    """b200_darts_normal into NaN-filled buffers -> (MM, M^H y)"""
    torch, dev, L = env
    nc = 2 * (2 * M_x + 1) * (2 * M_y + 1)
    rows = (2 * N_t + 1) * (2 * N_y + 1) * (2 * N_x + 1)
    x = _up(env, X)
    part = _nan(env, -(-rows // E.NORMAL_ROWS) * (nc * (nc + 1) // 2 + nc), torch.complex128)
    mm, mhy = _nan(env, nc * nc, torch.complex128), _nan(env, nc, torch.complex128)
    L.call("b200_darts_normal", x.data_ptr(), N_x, N_y, N_t, M_x, M_y, sx, sy, part.data_ptr(), mm.data_ptr(),
           mhy.data_ptr(), dev.stream_ptr())
    return mm.cpu().numpy().reshape(nc, nc), mhy.cpu().numpy()


def _synthesize(env, coef, ey, ex, m, n):
    torch, dev, L = env
    c, a, b = _up(env, coef), _up(env, ey), _up(env, ex)
    out = _nan(env, 2 * m * n, torch.float64)
    L.call("b200_darts_synthesize", c.data_ptr(), coef.shape[1], coef.shape[2], a.data_ptr(), b.data_ptr(), m, n,
           out.data_ptr(), dev.stream_ptr())
    return out.cpu().numpy().reshape(2, m, n)


def _check_normal(env, X, N_x, N_y, N_t, M_x, M_y, sx, sy, what):
    MM, Mhy = _normal(env, X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    assert not (np.isnan(MM).any() or np.isnan(Mhy).any()), f"{what}: NaN left in MM or M^H y"
    want_MM, want_Mhy = E.normal_restated(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    assert np.array_equal(MM.view(np.int64), want_MM.view(np.int64)), f"{what}: MM not bit-identical"
    assert np.array_equal(Mhy.view(np.int64), want_Mhy.view(np.int64)), f"{what}: M^H y not bit-identical"
    assert E.is_hermitian_bitwise(MM), what
    r = E.normal_ratio(MM, Mhy, E.normal_exact(X, N_x, N_y, N_t, M_x, M_y, sx, sy))
    print(f"{what}: normal error / bound = {r:.3e}")
    assert r <= 1.0, (what, r)


@pytest.mark.parametrize("case", E.SPECTRUM_CASES, ids=lambda c: c[0])
def test_spectrum_and_its_normal_equations_at_the_edges(env, case):
    name, T, m, n, N_x, N_y, N_t, M_x, M_y, kind, dtype = case
    R = E.frames(T, m, n, seed=len(name), kind=kind, dtype=dtype)
    X, tabs = _spectrum(env, R, N_x, N_y, N_t, M_x, M_y)
    assert not np.isnan(X).any(), f"{name}: NaN left in the spectrum"
    Xr, Xi, B = E.spectrum(R, *tabs)
    r = E.complex_ratio(X, Xr, Xi, B)
    print(f"{name}: spectrum error / bound = {r:.3e} (fx = {tabs[0].shape[0]})")
    assert r <= 1.0, (name, r)
    _check_normal(env, X, N_x, N_y, N_t, M_x, M_y, *E.normal_scales(T, m, n), name)


def test_large_spectrum_at_sampled_entries(env):
    """2048^2, T = 6, N_x = N_y = 200, M = 5: fx = 206, four frequency tiles; 8 kx (either side of
    the tile edges 64 and 128, 0 and the block's ends) x 8 ky x every kt"""
    from pysteps_b200 import _synthetic as syn
    T, m, n, N_x, N_y, N_t, M_x, M_y = 6, 2048, 2048, 200, 200, 4, 5, 5
    R = syn.rain_frames(m, n, T, seed=31, dx=3, dy=-2)
    X, tabs = _spectrum(env, R, N_x, N_y, N_t, M_x, M_y)
    assert tabs[0].shape[0] == 206 and not np.isnan(X).any()
    K = tabs[3]
    kx = K + np.array([-205, -129, -64, -1, 0, 63, 128, 205])
    ky = np.array([0, 15, 16, 31, 32, 205, 394, 410])
    Xr, Xi, B = E.spectrum(R, *tabs, kx=kx, ky=ky)
    r = E.complex_ratio(X[:, ky][:, :, kx], Xr, Xi, B)
    print(f"2048^2: spectrum error / bound = {r:.3e} at {Xr.size} entries")
    assert r <= 1.0, r


@pytest.mark.parametrize("case", E.NORMAL_CASES, ids=lambda c: c[0])
def test_normal_on_random_blocks(env, case):
    name, N_x, N_y, N_t, M_x, M_y = case
    X = E.random_block(N_x, N_y, N_t, M_x, M_y, seed=len(name))
    _check_normal(env, X, N_x, N_y, N_t, M_x, M_y, *E.normal_scales(4, 64, 96), name)


def test_normal_over_many_row_blocks(env):
    """N = (30, 30, 4), M = 5: 33 489 rows in 66 blocks, 29 645 pairs in 29 slabs.  Against the
    restatement at a sample of pairs: each slab's first and last, the diagonal, all of M^H y and
    2048 more (the whole restatement takes half a minute)"""
    N_x, N_y, N_t, M_x, M_y = 30, 30, 4, 5, 5
    X = E.random_block(N_x, N_y, N_t, M_x, M_y, seed=66)
    MM, Mhy = _normal(env, X, N_x, N_y, N_t, M_x, M_y, *E.normal_scales(6, 256, 256))
    assert not (np.isnan(MM).any() or np.isnan(Mhy).any())
    assert E.is_hermitian_bitwise(MM)
    nc = MM.shape[0]
    npairs = nc * (nc + 1) // 2 + nc
    q = np.arange(nc)
    slab = np.arange(0, npairs, 1024)
    sel = np.unique(np.concatenate([slab, np.minimum(slab + 1023, npairs - 1), q * (q + 1) // 2 + q,
                                    npairs - nc + q,
                                    np.random.default_rng(7).choice(npairs, 2048, replace=False)]))
    c, d, want = E.normal_restated(X, N_x, N_y, N_t, M_x, M_y, *E.normal_scales(6, 256, 256), sel=sel)
    got = np.where(d < nc, MM[c, np.minimum(d, nc - 1)], Mhy[c])
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


@pytest.mark.parametrize("shape", E.SYNTH_CASES, ids=lambda s: "x".join(map(str, s)))
def test_synthesis_within_the_bound(env, shape):
    h, w, m, n = shape
    coef, ey, ex = E.random_synthesis(h, w, m, n, seed=h * w + m)
    got = _synthesize(env, coef, ey, ex, m, n)
    assert not np.isnan(got).any()
    want, B = E.synthesize(coef, ey, ex, m, n)
    r = E._ratio(abs(E._ld(got) - want), B)
    print(f"{shape}: synthesis error / bound = {r:.3e}")
    assert r <= 1.0, r
    zero = _synthesize(env, np.zeros_like(coef), ey, ex, m, n)
    assert np.all(zero == 0)


def test_synthesis_of_colliding_coefficients(env):
    """M_x = 5, M_y = 2 on a 3 x 9 frame: fill_tables puts several coefficients on one wrapped index
    and the last write wins, as NumPy's fancy assignment in the reference's _fill does; the device
    field equals Re(ifft2) of that dense placement within the bound of the dense sum"""
    from pysteps_b200.motion import darts as dm
    M_x, M_y, m, n = 5, 2, 3, 9
    rng = np.random.default_rng(12)
    UV = rng.standard_normal((2, 2 * M_y + 1, 2 * M_x + 1)) + 1j * rng.standard_normal((2, 2 * M_y + 1, 2 * M_x + 1))
    rows, cols, ri, ci = dm.fill_tables(M_x, M_y, m, n)
    assert len(rows) < 2 * M_y + 1 and len(cols) < 2 * M_x + 1
    coef = np.zeros((2, len(rows), len(cols)), dtype=complex)
    coef[0][ri, ci] = UV[0]
    coef[1][ri, ci] = UV[1]
    got = _synthesize(env, coef, dm.twiddles(tuple(rows), m, 1), dm.twiddles(tuple(cols), n, 1), m, n)
    k_x, k_y = np.meshgrid(np.arange(-M_x, M_x + 1), np.arange(-M_y, M_y + 1))
    dense = np.zeros((2, m, n), dtype=complex)
    dense[0][k_y, k_x] = UV[0]
    dense[1][k_y, k_x] = UV[1]
    want, B = E.synthesize(dense, dm.twiddles(tuple(range(m)), m, 1), dm.twiddles(tuple(range(n)), n, 1), m, n)
    r = E._ratio(abs(E._ld(got) - want), B)
    print(f"colliding placement: synthesis error / bound = {r:.3e}")
    assert r <= 1.0, r


def test_synthesis_refuses_more_than_max_side_columns(env):
    torch, dev, L = env
    h, w, m, n = 1, 122, 1, 200
    coef, ey, ex = (_nan(env, k, torch.complex128) for k in (2 * h * w, h * m, w * n))
    out = _nan(env, 2 * m * n, torch.float64)
    with pytest.raises(RuntimeError, match=r"code 100001\).*B200_DARTS_MAX_SIDE"):
        L.call("b200_darts_synthesize", coef.data_ptr(), h, w, ey.data_ptr(), ex.data_ptr(), m, n, out.data_ptr(),
               dev.stream_ptr())
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
