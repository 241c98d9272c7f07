"""CPU test of the HOST logic of pysteps_b200.verification (argument checks, exceptions and messages,
warnings, returned types and dtypes, dict contents, the random draw of rankhist), with the entry
points of csrc/verification.cu emulated (tests/cpu_abi_verification.py).  Compared with the stored
reference outcomes, and with the live reference where it exists on randomised valid and invalid calls
and on dicts passed between the two."""
import os

import numpy as np
import pytest

import cpu_abi_verification
from verification_cases import Goldens, golden_calls, matches_golden, reference, run_call, same_outcome

GOLDEN = Goldens(os.path.join(os.path.dirname(__file__), "golden", "verification_golden.npz"))
CALLS = golden_calls()


def _ours():
    from pysteps_b200.verification import ensscores, probscores
    return {"probscores": probscores, "ensscores": ensscores}


@pytest.mark.parametrize("i", range(len(CALLS)), ids=[c[0] for c in CALLS])
def test_golden_calls_through_the_host(i):
    key, mod, fn, args, seed = CALLS[i]
    with cpu_abi_verification.emulated():
        out, warned, nxt = run_call(_ours()[mod], fn, args, seed)
    assert not matches_golden(GOLDEN, key, out, warned, nxt), (key, matches_golden(GOLDEN, key, out, warned, nxt))


@pytest.fixture(scope="module")
def ref():
    r = reference()
    if r is None:
        pytest.skip("the reference is not present")
    return {"probscores": r[0], "ensscores": r[1]}


def _field(rng, shape, dtype):
    X = np.where(rng.random(shape) < 0.4, 0.0, rng.gamma(0.8, 2.0, shape))
    if rng.random() < 0.5:
        u = rng.random(shape)
        X[u < 0.1] = np.nan
        X[(u >= 0.1) & (u < 0.13)] = np.inf
    if rng.random() < 0.05:
        X[...] = np.nan
    if dtype in (np.int64,):
        return np.nan_to_num(X, posinf=9).astype(dtype)
    return X.astype(dtype)


def _dtype(rng):
    return np.int64 if rng.random() < 0.06 else [np.float32, np.float64][int(rng.integers(0, 2))]


def _xmin(rng, allow_none):
    v = float(rng.choice([0.0, 0.1, 0.5, 1.0, 2.5]))
    kinds = [v, np.float64(v), np.float32(v), int(v), np.array(v)] + ([None] if allow_none else [])
    return kinds[int(rng.integers(0, len(kinds)))]


def _shapes(rng):
    """(member shape, observation shape): mostly matching, sometimes not"""
    m = tuple(int(rng.integers(0 if rng.random() < 0.05 else 1, 7)) for _ in range(int(rng.integers(1, 4))))
    r = rng.random()
    if r < 0.75:
        return m, m
    if r < 0.85:
        return m, (int(np.prod(m)),)
    if r < 0.9:
        return m, (1,)
    return m, tuple(int(rng.integers(0, 5)) for _ in range(int(rng.integers(0, 3))))


def _random_call(rng):
    """(module, function, args, seed)"""
    which = int(rng.integers(0, 8))
    fshape, oshape = _shapes(rng)
    if which in (0, 1, 2, 3):  # CRPS / rankhist, wrapper or accumulation
        k = int(rng.choice([0, 1, 2, 3, 7, 9])) if rng.random() < 0.95 else 600
        X_f = _field(rng, (k,) + fshape if rng.random() < 0.97 else fshape, _dtype(rng))
        X_o = _field(rng, oshape, _dtype(rng))
        if which == 0:
            return "probscores", "CRPS", (X_f, X_o), None
        if which == 1:
            return "probscores", "CRPS_accum", ((), X_f, X_o), None
        xm = _xmin(rng, True)
        if rng.random() < 0.3 and X_f.ndim:
            X_o = X_f[int(rng.integers(0, X_f.shape[0]))].copy() if X_f.shape[0] else X_o  # ties
        if which == 2:
            return "ensscores", "rankhist", (X_f, X_o, xm, bool(rng.random() < 0.5)), int(rng.integers(0, 99))
        kd = X_f.shape[0] if X_f.ndim and rng.random() < 0.9 else 3
        return "ensscores", "rankhist_accum", ((kd, xm), X_f, X_o), int(rng.integers(0, 99))
    P = (rng.integers(0, 11, fshape) / 10.0).astype(_dtype(rng) if rng.random() < 0.9 else np.float32)
    if rng.random() < 0.3:
        P = P.astype(np.float64)
        P[rng.random(fshape) < 0.1] = np.nan
    X_o = _field(rng, oshape, _dtype(rng))
    xm = _xmin(rng, False)
    n = [1, 2, 3, 10, 0, 10.0, -1][int(rng.integers(0, 7))]
    if which in (4, 5):
        mc = [0, 1, 3, 10][int(rng.integers(0, 4))]
        if which == 4:
            return "probscores", "reldiag", (P, X_o, xm, n, mc), None
        return "probscores", "reldiag_accum", ((xm, n, mc), P, X_o), None
    if which == 6:
        return "probscores", "ROC_curve", (P, X_o, xm, n, bool(rng.random() < 0.5)), None
    return "probscores", "ROC_curve_accum", ((xm, n), P, X_o), None


def test_randomised_calls_against_the_reference(ref):
    rng = np.random.default_rng(2024)
    ours = _ours()
    compared = refused = 0
    for t in range(500):
        mod, fn, args, seed = _random_call(rng)
        seed = t if seed is None else seed  # every call from a known state, so the state after it can be compared
        want = run_call(ref[mod], fn, args, seed)
        with cpu_abi_verification.emulated():
            got = run_call(ours[mod], fn, args, seed)
        if isinstance(got[0], NotImplementedError):
            refused += 1
            continue
        compared += 1
        assert same_outcome(got[0], want[0]), (t, fn, got[0], want[0])
        assert got[1] == want[1], (t, fn, got[1], want[1])
        assert got[2] == want[2], (t, fn, "the random state after the call differs")
    assert compared >= 400 and refused < 100, (compared, refused)


def test_empty_broadcast_shapes_as_the_reference(ref):
    ours = _ours()
    for fn, args in (("reldiag", (np.zeros(0), np.ones(1), 0.5)), ("ROC_curve", (np.zeros(0), np.ones(1), 0.5)),
                     ("reldiag", (np.ones(1), np.zeros(0), 0.5)), ("CRPS", (np.zeros((3, 0)), np.ones(1)))):
        want = run_call(ref["probscores"], fn, args, None)
        with cpu_abi_verification.emulated():
            got = run_call(ours["probscores"], fn, args, None)
        assert same_outcome(got[0], want[0]) and got[1] == want[1], (fn, got, want)


def test_dicts_pass_between_the_reference_and_this_package(ref):
    ours = _ours()
    rng = np.random.default_rng(7)
    X_f = _field(rng, (6, 20, 30), np.float32)
    X_o = _field(rng, (20, 30), np.float64)
    P = (rng.integers(0, 7, (20, 30)) / 6.0)
    plans = (("probscores", "CRPS", (), (X_f, X_o), ()), ("ensscores", "rankhist", (6, 0.1), (X_f, X_o), ()),
             ("probscores", "reldiag", (0.5, 10, 3), (P, X_o), ()), ("probscores", "ROC_curve", (0.5, 10), (P, X_o),
                                                                        (True,)))
    for mod, name, init_args, data, comp_args in plans:
        init, accum, compute = name + "_init", name + "_accum", name + "_compute"
        for first, second in ((ref, ours), (ours, ref)):
            np.random.seed(5)
            d = getattr(first[mod], init)(*init_args)
            with cpu_abi_verification.emulated():
                getattr(ours[mod], accum)(d, *data)
            getattr(ref[mod], accum)(d, *data)
            got = run_call(second[mod], compute, (d,) + comp_args, None)
            np.random.seed(5)
            w = getattr(ref[mod], init)(*init_args)
            getattr(ref[mod], accum)(w, *data)
            getattr(ref[mod], accum)(w, *data)
            want = run_call(ref[mod], compute, (w,) + comp_args, None)
            assert same_outcome(d, w), name
            assert same_outcome(got[0], want[0]) and got[1] == want[1], name
