"""CPU test of the HOST logic of pysteps_b200.motion.darts (argument checks and their order, the
fft_method lookup, NumPy's IndexError for short axes, verbose output, dtypes, the solve and the
return structure), with the three entry points of csrc/darts.cu emulated by the oracle
(tests/cpu_abi_darts.py).  Compared with the live reference on randomised valid and invalid calls."""
import contextlib
import io
import re

import numpy as np
import pytest

import cpu_abi_darts
from pysteps_b200 import _synthetic as syn


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.motion.darts")


def _run(fn, R, kw):
    """-> (result or exception, stdout with the timings masked)"""
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        try:
            out = fn(R, **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            out = e
    return out, re.sub(r"\d+\.\d+(e-?\d+)?", "<t>", buf.getvalue())


def _same_outcome(got, want, bar):
    if isinstance(want, Exception):
        assert type(got) is type(want) and str(got) == str(want), (got, want)
        return
    assert isinstance(got, np.ndarray) and got.dtype == want.dtype and got.shape == want.shape, (got, want)
    assert np.abs(got - want).max() <= bar * max(np.abs(want).max(), 0.0), np.abs(got - want).max()


def _random_call(rng):
    kind = int(rng.integers(0, 14))
    m, n = (int(k) for k in rng.integers(20, 72, 2))
    T = int(rng.integers(3, 8))
    N_x, N_y = (int(k) for k in rng.integers(2, 40, 2))
    kw = dict(N_x=N_x, N_y=N_y, N_t=int(rng.integers(0, T - 1)), M_x=int(rng.integers(0, 3)),
              M_y=int(rng.integers(0, 3)), verbose=bool(rng.integers(2)))
    R = syn.rain_frames(m, n, T, seed=int(rng.integers(1000)), dx=int(rng.integers(-3, 4)), dy=int(rng.integers(-3, 4)))
    if kind == 0:
        return R[0], kw                                       # 2-D
    if kind == 1:
        kw["N_t"] = T - 1 - int(rng.integers(0, 2))           # N_t >= T - 1
    if kind == 2:
        kw["output_type"] = "grid"
    if kind == 3:
        R[int(rng.integers(T)), 3, 4] = [np.nan, np.inf][int(rng.integers(2))]
    if kind == 4:
        kw["fft_method"] = ["FFTW", "sqrt", "none", None, "SciPy", "pyfftw"][int(rng.integers(6))]
    if kind == 5:
        kw.pop("N_x"), kw.pop("N_y")                          # defaults: IndexError on these frames
    if kind == 6:
        kw["N_y"] = m - int(rng.integers(0, 2))                # the y-vector loop fails
    if kind == 7:
        kw["M_x"] = n - kw["N_x"] + int(rng.integers(0, 2))   # the H-matrix loop fails
        kw["M_x"] = min(kw["M_x"], 5)
    if kind == 8:
        kw["lsq_method"] = 1
    if kind == 9:
        kw["output_type"] = "spectral"
    if kind == 10:
        R = R.astype(np.float32)
    if kind == 11:
        R = np.full_like(R, 1.5)
    if kind == 12:
        kw["unused_option"] = 3
    return R, kw


def test_random_calls_match_the_live_reference():
    ref = _reference()
    from pysteps_b200.motion import get_method
    ours = get_method("darts")
    rng = np.random.default_rng(2025)
    for _ in range(60):
        R, kw = _random_call(rng)
        # "pyfftw" names the same DFT on the device, with or without pyfftw (DESIGN.md section 4)
        ref_kw = dict(kw, fft_method="numpy") if kw.get("fft_method") == "pyfftw" else kw
        want, want_out = _run(ref.DARTS, R, ref_kw)
        with cpu_abi_darts.emulated():
            got, got_out = _run(ours, R, kw)
        bar = 1e-6 if R.dtype == np.float32 else 1e-9
        _same_outcome(got, want, bar)
        assert got_out == want_out, (kw, got_out, want_out)


@pytest.mark.parametrize("shape,kw", [((6, 52, 60), {}), ((6, 60, 50), {}), ((6, 60, 60), dict(N_x=57, M_x=3)),
                                      ((6, 60, 60), dict(N_y=58, M_y=2)), ((6, 8, 9), dict(N_x=4, N_y=4, M_x=5))])
def test_short_axes_raise_numpy_index_error(shape, kw):
    ref = _reference()
    from pysteps_b200.motion.darts import DARTS
    R = np.random.default_rng(1).standard_normal(shape)
    kw = dict(kw, verbose=True)
    want, want_out = _run(ref.DARTS, R, kw)
    with cpu_abi_darts.emulated():
        got, got_out = _run(DARTS, R, kw)
    assert isinstance(want, IndexError)
    _same_outcome(got, want, 0.0)
    assert got_out == want_out


def test_fft_method_errors_and_check_order():
    ref = _reference()
    from pysteps_b200.motion.darts import DARTS
    R = syn.rain_frames(60, 60, 6, seed=2)
    bad = R.copy()
    bad[1, 2, 3] = np.nan
    calls = [(R, dict(fft_method="unknown")), (R, dict(fft_method="sqrt")), (R, dict(fft_method=3)),
             (bad, dict(fft_method="unknown")), (bad, dict(output_type="x")), (bad, dict(N_t=5, output_type="x")),
             (np.zeros((2, 2, 5, 5)), dict(N_t=9)), (R, dict(N_x=70, output_type="x"))]
    for R_, kw in calls:
        kw = dict(kw, verbose=True, N_x=kw.get("N_x", 20), N_y=20)
        want, want_out = _run(ref.DARTS, R_, kw)
        with cpu_abi_darts.emulated():
            got, got_out = _run(DARTS, R_, kw)
        assert isinstance(want, Exception), kw
        _same_outcome(got, want, 0.0)
        assert got_out == want_out


def test_masked_nan_under_the_mask_reaches_the_solve():
    ref = _reference()
    from darts_cases import build_case
    from pysteps_b200.motion.darts import DARTS
    R, kw = build_case("masked_nan_128x96")
    for lsq in (1, 2):
        want, _ = _run(ref.DARTS, R, dict(kw, lsq_method=lsq))
        with cpu_abi_darts.emulated():
            got, _ = _run(DARTS, R, dict(kw, lsq_method=lsq))
        assert isinstance(want, np.linalg.LinAlgError)
        _same_outcome(got, want, 0.0)


def test_integer_frames_and_too_many_unknowns_are_refused():
    from pysteps_b200.motion.darts import DARTS
    with cpu_abi_darts.emulated():
        with pytest.raises(NotImplementedError, match="int64"):
            DARTS(np.ones((6, 64, 64), dtype=np.int64), verbose=False)
        with pytest.raises(NotImplementedError, match="M_x, M_y <= 5"):
            DARTS(np.ones((6, 64, 64)), verbose=False, N_x=5, N_y=5, M_x=6, M_y=5)
