"""CPU test of the HOST logic of pysteps_b200.nowcasts.lagrangian_probability (argument flow,
exceptions and their order, the threshold rules, extrapolation methods, dtypes and shapes), with the
entry point of csrc/probability.cu and the extrapolator emulated by the oracle
(tests/cpu_abi_probability.py).  Compared with the live reference where it exists, on randomised
valid and invalid calls."""
import os

import numpy as np
import pytest

import cpu_abi_probability
from oracle import probability as ora
from probability_cases import CASES, LARGE, build_case
from pysteps_b200 import _synthetic as syn

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "probability_golden.npz")
BOUND = 1e-6


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.nowcasts.lagrangian_probability")


def _run(fn, args, kw):
    try:
        return fn(*args, **kw)
    except Exception as e:  # noqa: BLE001 -- the exception is the result
        return e


def _same_outcome(got, want, what):
    if isinstance(want, Exception):
        # first line: the lists of available extrapolators differ by this package's "_b200" aliases
        assert type(got) is type(want) and str(got).split("\n")[0] == str(want).split("\n")[0], (what, got, want)
        return
    assert isinstance(got, np.ndarray) and got.dtype == want.dtype == np.float64 and got.shape == want.shape, what
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    if (~nan).any():
        assert np.abs(got[~nan] - want[~nan]).max() <= BOUND, what


@pytest.mark.parametrize("name", [c for c in CASES if c not in LARGE])
def test_golden_cases_through_the_host(name):
    from pysteps_b200.nowcasts.lagrangian_probability import forecast
    args, kw = build_case(name)
    with cpu_abi_probability.emulated():
        got = forecast(*args, **kw)
    want = ora.forecast(*args, **kw)
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and got.shape == want.shape
    assert np.array_equal(got, want, equal_nan=True)
    _same_outcome(got, np.load(GOLDEN)[name + "/out"], name)


def _random_call(rng):
    """(args, kwargs) of one call, valid or not"""
    kind = int(rng.integers(0, 20))
    m, n = (int(k) for k in rng.integers(8, 40, 2))
    P = syn.rain_field(m, n, int(rng.integers(1000)))
    V = syn.velocity_field(m, n, int(rng.integers(1000)))
    T = int(rng.integers(1, 5))
    thr = float(rng.choice([0.5, 5.0, 12.0]))
    kw = {}
    if kind == 0:
        T = int(rng.integers(-2, 1))                                  # 0 or negative
    elif kind == 1:
        T = np.arange(1, 3) if rng.integers(2) else 2.0              # an array or a float
    elif kind == 2:
        P = P[None]                                                   # 3-D precip
    elif kind == 3:
        V = V[0]                                                      # 2-D velocity
    elif kind == 4:
        V = V[:, :-1]                                                 # shape mismatch
    elif kind == 5:
        T = [1.0, 3.0, 2.0]                                           # unsorted list
    elif kind == 6:
        kw["extrap_method"] = rng.choice(["nope", None, "none"])
    elif kind == 7:
        kw["slope"] = -float(rng.integers(1, 4))                      # negative diameters
    elif kind == 8:
        V = V.copy()
        V[0, 0, 0] = np.nan                                           # refused: precip is finite
    elif kind == 9:
        thr = None
    elif kind == 10:
        kw["extrap_kwargs"] = {"return_displacement": True}
        T = 2 if rng.integers(2) else 3
    elif kind == 11:
        P = syn.nan_disc(P, 0.3)
        V = V.copy()
        V[1, 2, 3] = np.inf                                           # allowed: precip has NaN
    elif kind == 12:
        T = sorted(float(t) for t in rng.uniform(0, 3, 4))
        kw["slope"] = float(rng.uniform(0, 6))
    elif kind == 13:
        P = syn.nan_disc(P, 0.25).astype(np.float32)
        thr = float(rng.choice([3e8, np.inf, -np.inf, np.nan]))
    elif kind == 14:
        kw["extrap_method"] = "Eulerian"
        P = syn.nan_disc(P, 0.2)
    elif kind == 15:
        kw["extrap_kwargs"] = {"vel_timestep": 2, "interp_order": int(rng.choice([0, 1, 3])), "outval": 0.0}
    elif kind == 16:
        T = True
    elif kind == 17:
        kw["extrap_method"] = "SemiLagrangian"
        kw["extrap_kwargs"] = {"allow_nonfinite_values": False}
        P = syn.nan_disc(P, 0.2)
    elif kind == 18:
        kw["slope"] = 0
        P = P.astype(np.float32)
    else:
        T = [0.05, 0.5, 1.0]
        kw["slope"] = 40                                              # kernels larger than the frame
    return (P, V, T, thr), kw


def test_random_calls_match_the_live_reference():
    ref = _reference()
    from pysteps_b200.nowcasts import get_method
    ours = get_method("probability")
    rng = np.random.default_rng(2026)
    for i in range(80):
        args, kw = _random_call(rng)
        want = _run(ref.forecast, args, kw)
        with cpu_abi_probability.emulated():
            got = _run(ours, args, kw)
        _same_outcome(got, want, (i, kw))


def test_integer_fields_are_refused():
    from pysteps_b200.nowcasts.lagrangian_probability import forecast
    with cpu_abi_probability.emulated():
        with pytest.raises(NotImplementedError, match="int64"):
            forecast(np.ones((8, 8), dtype=np.int64), np.zeros((2, 8, 8)), 2, 1.0)
