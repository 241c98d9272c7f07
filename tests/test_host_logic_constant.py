"""CPU test of the HOST logic of pysteps_b200.motion.constant (shape and frame handling, dtypes,
MaskedArray input, the reference's RuntimeWarnings, return structure), with the two entry points of
csrc/constant.cu emulated by the oracle (tests/cpu_abi_constant.py).  Compared with the live reference where
it exists, on randomised valid and invalid calls."""
import os
import warnings

import numpy as np
import pytest

import cpu_abi_constant
from constant_cases import CASES, LARGE, ORDER_DECIDED, build_case

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "constant_golden.npz")


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.motion.constant")


def _run(fn, R):
    """-> (result or exception, [(category, message), ...]) with every warning recorded"""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            out = fn(R)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            out = e
    return out, [(x.category, str(x.message)) for x in w]


def _same_outcome(got, want):
    if isinstance(want, Exception):
        assert type(got) is type(want) and str(got) == str(want), (got, want)
        return
    assert isinstance(got, np.ndarray) and got.dtype == want.dtype == np.float64 and got.shape == want.shape
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


@pytest.mark.parametrize("name", [c for c in CASES if c not in LARGE])
def test_golden_cases_through_the_host(name):
    from pysteps_b200.motion.constant import constant
    from oracle import constant as ora
    g = np.load(GOLDEN)
    R = build_case(name)
    m, n = R.shape[1:]
    with cpu_abi_constant.emulated(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = constant(R)
        want = ora.constant(R)
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and got.shape == (2, m, n)
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    x = g[name + "/x"]
    ref = np.stack([-x[0] * np.ones((m, n)), -x[1] * np.ones((m, n))])
    if name not in ORDER_DECIDED:  # (see constant_cases.py)
        assert np.array_equal(got.view(np.int64), ref.view(np.int64))


def _random_call(rng):
    kind = rng.integers(0, 12)
    m, n = (int(k) for k in rng.integers(1, 24, 2))
    T = int(rng.integers(2, 4))
    if kind == 0:
        return np.zeros((m, n))                          # 2-D
    if kind == 1:
        return np.zeros((2, 2, m, n))                    # 4-D
    if kind == 2:
        return np.zeros((int(rng.integers(0, 2)), m, n))  # fewer than two frames
    if kind == 3:
        return np.zeros((2, 0, n)) if rng.integers(2) else np.zeros((2, m, 0))
    if kind == 4:
        return np.ones((2, m, n), np.float16)
    if kind == 5:
        R = np.full((T, m, n), np.nan)
        R[:, int(rng.integers(m)), int(rng.integers(n))] = 1.0
        return R
    if kind == 6:
        return np.full((T, m, n), 0.1)
    R = rng.standard_normal((T, m, n)) * 3.0
    if kind in (7, 8):
        R[rng.random((T, m, n)) < 0.2] = np.nan
    if kind == 8:
        R[-1] = np.nan
    if kind == 9:
        R = np.ma.MaskedArray(R, mask=rng.random((T, m, n)) < 0.3)
    if kind == 10:
        R = R.astype(np.float32)
    return R


def test_random_calls_match_the_live_reference():
    ref = _reference()
    from pysteps_b200.motion import get_method
    ours = get_method("constant")
    rng = np.random.default_rng(2024)
    for _ in range(40):
        R = _random_call(rng)
        want, want_w = _run(ref.constant, R)
        with cpu_abi_constant.emulated():
            got, got_w = _run(ours, R)
        _same_outcome(got, want)
        assert got_w == want_w


def test_argument_errors_match_the_live_reference():
    ref = _reference()
    from pysteps_b200.motion.constant import constant
    for R in ([[[1.0]]], np.float64(1.0), np.zeros(3), np.zeros((1, 4, 4)), np.zeros((0, 4, 4))):
        want, _ = _run(ref.constant, R)
        with cpu_abi_constant.emulated():
            got, _ = _run(constant, R)
        _same_outcome(got, want)


def test_errstate_raise_acts_on_the_warnings():
    ref = _reference()
    from pysteps_b200.motion.constant import constant
    R = np.full((2, 6, 5), np.nan)
    with np.errstate(all="raise"):
        want, _ = _run(ref.constant, R)
        with cpu_abi_constant.emulated():
            got, _ = _run(constant, R)
    assert isinstance(want, FloatingPointError) and type(got) is type(want) and str(got) == str(want)


def test_kwargs_are_ignored_and_integer_frames_are_refused():
    from pysteps_b200.motion.constant import constant
    R = build_case("odd_width_31x97")
    with cpu_abi_constant.emulated():
        assert np.array_equal(constant(R, verbose=True, anything=3), constant(R))
        with pytest.raises(NotImplementedError, match="int64"):
            constant(np.ones((2, 4, 4), dtype=np.int64))
