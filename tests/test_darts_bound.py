"""CPU: the extended-precision references and bounds of darts_exact.py.  The float64 oracle
(oracle/darts.py) and the bit-level restatement of darts_normal_kernel lie within the bounds at the
kernels' edge cases; the spectrum bound is not vacuous on a smooth rain case; and the comparison
fails restatements carrying the bugs it exists to catch (a dropped conjugate, a transposed twiddle
read, a dropped partial row block, a second frequency tile offset by one)."""
import numpy as np
import pytest

import darts_exact as E
from oracle import darts as ora
from pysteps_b200.motion import darts as dm


def _case(name, cases):
    return next(c for c in cases if c[0] == name)


def _spectrum_inputs(name):
    _, T, m, n, N_x, N_y, N_t, M_x, M_y, kind, dtype = _case(name, E.SPECTRUM_CASES)
    R = E.frames(T, m, n, seed=len(name), kind=kind, dtype=dtype)
    return R, dm.spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y)


@pytest.mark.parametrize("name", [c[0] for c in E.SPECTRUM_CASES])
def test_oracle_spectrum_is_within_the_bound(name):
    R, (tw_x, tw_y, tw_t, K) = _spectrum_inputs(name)
    Xr, Xi, B = E.spectrum(R, tw_x, tw_y, tw_t, K)
    got = ora.spectrum_from_tables(R, tw_x, tw_y, tw_t, K)
    assert got.shape == Xr.shape
    r = E.complex_ratio(got, Xr, Xi, B)
    print(f"{name}: oracle spectrum error / bound = {r:.3e}")
    assert r <= 1.0


@pytest.mark.parametrize("name", [c[0] for c in E.NORMAL_CASES])
def test_normal_restatement_and_oracle_are_within_the_bound(name):
    _, N_x, N_y, N_t, M_x, M_y = _case(name, E.NORMAL_CASES)
    X = E.random_block(N_x, N_y, N_t, M_x, M_y, seed=len(name))
    sx, sy = E.normal_scales(4, 64, 96)
    ex = E.normal_exact(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    MM, Mhy = E.normal_restated(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    assert E.is_hermitian_bitwise(MM)
    r = E.normal_ratio(MM, Mhy, ex)
    oMM, oMhy = ora.normal(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    ro = E.normal_ratio(oMM, oMhy, ex)
    print(f"{name}: restatement {r:.3e}, oracle {ro:.3e} of the bound")
    assert r <= 1.0 and ro <= 1.0


@pytest.mark.parametrize("name", ["fx66", "alias_odd101", "t2_nt0"])
def test_normal_on_spectra_is_within_the_bound(name):
    R, (tw_x, tw_y, tw_t, K) = _spectrum_inputs(name)
    _, T, m, n, N_x, N_y, N_t, M_x, M_y, _, _ = _case(name, E.SPECTRUM_CASES)
    X = ora.spectrum_from_tables(R, tw_x, tw_y, tw_t, K)
    sx, sy = E.normal_scales(T, m, n)
    ex = E.normal_exact(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    r = E.normal_ratio(*E.normal_restated(X, N_x, N_y, N_t, M_x, M_y, sx, sy), ex)
    ro = E.normal_ratio(*ora.normal(X, N_x, N_y, N_t, M_x, M_y, sx, sy), ex)
    print(f"{name}: restatement {r:.3e}, oracle {ro:.3e} of the bound")
    assert r <= 1.0 and ro <= 1.0


@pytest.mark.parametrize("shape", E.SYNTH_CASES, ids=lambda s: "x".join(map(str, s)))
def test_oracle_synthesis_is_within_the_bound(shape):
    h, w, m, n = shape
    coef, ey, ex = E.random_synthesis(h, w, m, n, seed=h * w + m)
    want, B = E.synthesize(coef, ey, ex, m, n)
    r = E._ratio(abs(E._ld(ora.synthesize(coef, ey, ex, m, n)) - want), B)
    print(f"{shape}: oracle synthesis error / bound = {r:.3e}")
    assert r <= 1.0


def _median_bound_over_entries(R, N_x, N_y, N_t, M_x, M_y):
    T, m, n = R.shape
    Xr, Xi, B = E.spectrum(R, *dm.spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y))
    return float(np.median(B / np.asarray(np.sqrt(Xr * Xr + Xi * Xi), np.float64)))


def test_spectrum_bound_is_not_vacuous():
    """The bound is gamma * sum |frames - c0| at every entry (|twiddle| = 1), so bound / |X| grows
    as the spectrum falls off inside the block.  On a smooth rain cell (a Gaussian moving 4 px per
    frame) at a small block its median is below 1e-12; on the rain frames of the golden case
    shift_256_f64 at DARTS's default block (N = 50, M = 2) below 1e-9."""
    from darts_cases import build_case
    y, x = np.mgrid[0:128, 0:128].astype(np.float64)
    cell = np.stack([20.0 * np.exp(-((y - 60 - 4 * t) ** 2 + (x - 64 + 4 * t) ** 2) / (2 * 8.0 ** 2))
                     for t in range(4)])
    smooth = _median_bound_over_entries(cell, 2, 2, 1, 1, 1)
    rain = _median_bound_over_entries(build_case("shift_256_f64")[0], 50, 50, 4, 2, 2)
    print(f"median bound / |X|: smooth cell {smooth:.3e}, rain at the default block {rain:.3e}")
    assert smooth < 1e-12 and rain < 1e-9


# ---- the comparison catches the bugs it exists to find ----------------------------------------
def _no_conjugate(R, tw_x, tw_y, tw_t, K):
    """oracle.spectrum_from_tables without the conjugate on aliased frequencies"""
    T, m, n = R.shape
    rows = R.reshape(T * m, n).astype(np.float64)
    rows = rows - rows[0, 0]
    P = (rows @ tw_x.real.T) + 1j * (rows @ tw_x.imag.T)
    f, _ = E.x_selection(K, n)
    Q = np.tensordot(tw_t, P.reshape(T, m, -1)[:, :, f], axes=(1, 0))
    return np.matmul(tw_y[None], Q)


def _transposed_read(tw_x):
    """tw[x, f] read for tw[f, x]: the flat table indexed x * fx + f"""
    fx, n = tw_x.shape
    f, x = np.meshgrid(np.arange(fx), np.arange(n), indexing="ij")
    return tw_x.ravel()[(x * fx + f) % tw_x.size]


def _second_tile_offset(tw_x):
    """frequencies f >= XF computed with row f + 1 (zero past the table), as a tile at f0 + 1 would"""
    out = tw_x.copy()
    fx = tw_x.shape[0]
    out[E.XF:fx - 1] = tw_x[E.XF + 1:]
    out[fx - 1] = 0
    return out


@pytest.mark.parametrize("mutation,name", [("dropped_conjugate", "alias_odd101"),
                                           ("dropped_conjugate", "alias_even96"),
                                           ("transposed_table", "fx66"),
                                           ("second_tile_offset", "fx66"),
                                           ("second_tile_offset", "fx129")])
def test_spectrum_mutation_fails_the_bound(mutation, name):
    R, (tw_x, tw_y, tw_t, K) = _spectrum_inputs(name)
    assert tw_x.shape[0] != tw_x.shape[1]
    Xr, Xi, B = E.spectrum(R, tw_x, tw_y, tw_t, K)
    if mutation == "dropped_conjugate":
        assert E.x_selection(K, R.shape[2])[1].any()
        bad = _no_conjugate(R, tw_x, tw_y, tw_t, K)
    else:
        assert tw_x.shape[0] > E.XF
        mutated = _transposed_read(tw_x) if mutation == "transposed_table" else _second_tile_offset(tw_x)
        bad = ora.spectrum_from_tables(R, mutated, tw_y, tw_t, K)
    r = E.complex_ratio(bad, Xr, Xi, B)
    print(f"{mutation} on {name}: error / bound = {r:.3e}")
    assert r > 1.0


@pytest.mark.parametrize("name", ["rows513_m55", "rows513_m21"])
def test_dropped_partial_block_fails_the_bound(name):
    _, N_x, N_y, N_t, M_x, M_y = _case(name, E.NORMAL_CASES)
    X = E.random_block(N_x, N_y, N_t, M_x, M_y, seed=len(name))
    sx, sy = E.normal_scales(4, 64, 96)
    ex = E.normal_exact(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    r = E.normal_ratio(*E.normal_restated(X, N_x, N_y, N_t, M_x, M_y, sx, sy, drop_last_partial=True), ex)
    print(f"{name} without its last partial block: error / bound = {r:.3e}")
    assert r > 1.0
