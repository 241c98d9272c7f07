"""CPU test of the HOST logic of pysteps_b200.postprocessing.ensemblestats (argument checks, exceptions,
warnings, threshold dtypes, shapes, dtypes and the random draw of banddepth), with the entry points
of csrc/ensemblestats.cu emulated by the oracle (tests/cpu_abi_ensemblestats.py).  Compared with the
stored reference outputs and warnings, and with the live reference where it exists, on randomised
valid and invalid calls."""
import os
import warnings

import numpy as np
import pytest

import cpu_abi_ensemblestats
from conftest import bits_equal
from ensemblestats_cases import CASES, LARGE, build_case, seed_of
from test_oracle_ensemblestats import check_golden

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ensemblestats_golden.npz")


def _ours(fn):
    from pysteps_b200.postprocessing import ensemblestats
    return getattr(ensemblestats, fn)


def _outcome(fn, args, kw, seed=None):
    """(result or exception, ["Category: message", ...], the next random draw)"""
    if seed is not None:
        np.random.seed(seed)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            out = fn(*args, **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            out = e
    return out, [f"{x.category.__name__}: {x.message}" for x in w], np.random.random()


@pytest.mark.parametrize("name", [c for c in CASES if c not in LARGE])
def test_golden_cases_through_the_host(name):
    fn, args, kw = build_case(name)
    seed = seed_of(name) if fn == "banddepth" else None
    with cpu_abi_ensemblestats.emulated():
        got, warned, nxt = _outcome(_ours(fn), args, kw, seed)
    assert isinstance(got, np.ndarray), got
    check_golden(name, got)
    g = np.load(GOLDEN)
    assert warned == list(g[name + "/warnings"]), name
    if fn == "banddepth":
        assert nxt == g[name + "/next"], "the random state after the call differs from the reference's"


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.postprocessing.ensemblestats")


def _random_X(rng, ndim, dtype):
    k = int(rng.choice([0, 1, 2, 3, 7]))
    shape = (k,) + tuple(int(rng.integers(0 if rng.random() < 0.05 else 1, 6)) for _ in range(ndim - 1))
    X = np.where(rng.random(shape) < 0.4, 0.0, rng.gamma(0.8, 2.0, shape))
    u = rng.random(shape)
    if rng.random() < 0.5:
        X[u < 0.1] = np.nan
        X[(u >= 0.1) & (u < 0.13)] = np.inf
        X[(u >= 0.13) & (u < 0.16)] = -np.inf
    if rng.random() < 0.1:
        X[:] = np.nan
    if dtype in (np.int64, np.bool_):
        return np.nan_to_num(X, posinf=9, neginf=-9).astype(dtype)
    return X.astype(dtype)


def _random_threshold(rng):
    v = float(rng.choice([0.0, 0.5, 1.0, 2.5, float(np.float32(0.1)) + 1e-12, np.nan]))
    kind = int(rng.integers(0, 5))
    return [v, np.float64(v), np.float32(v), int(v) if np.isfinite(v) else v, np.array(v)][kind]


def _random_call(rng):
    """(function name, args, kwargs, unsupported): one call, valid or not; `unsupported` marks the
    inputs this package declines with NotImplementedError"""
    fn = ["mean", "excprob", "banddepth"][int(rng.integers(0, 3))]
    dtype = [np.float32, np.float64, np.float64, np.float32, np.int64, np.bool_][int(rng.integers(0, 6))]
    ndim = int(rng.integers(1, 6))
    X = _random_X(rng, ndim, dtype)
    unsupported = dtype in (np.int64, np.bool_)
    if fn == "mean":
        kw = {}
        if rng.random() < 0.5:
            kw["ignore_nan"] = bool(rng.random() < 0.5)
        if rng.random() < 0.5:
            kw["X_thr"] = _random_threshold(rng)
        unsupported = unsupported and ndim in (2, 3)
        return fn, (X,), kw, unsupported
    if fn == "excprob":
        kind = int(rng.integers(0, 6))
        if kind == 0:
            thr = _random_threshold(rng)
        elif kind == 1:
            thr = [float(t) for t in rng.random(int(rng.integers(1, 11))) * 3]
        elif kind == 2:
            thr = rng.random(int(rng.integers(1, 4))) * 3
        elif kind == 3:
            thr = []
        elif kind == 4:
            thr = np.array(0.5)
        else:
            thr = (np.float32(0.5), 1, 2.0)
        kw = {"ignore_nan": bool(rng.random() < 0.5)} if rng.random() < 0.7 else {}
        unsupported = unsupported and ndim >= 3 and kind not in (3, 4)
        return fn, (X, thr), kw, unsupported
    kw = {}
    if rng.random() < 0.4:
        kw["thr"] = _random_threshold(rng)
    if rng.random() < 0.4:
        kw["norm"] = True
    unsupported = unsupported or ndim < 2
    return fn, (X,), kw, unsupported


def _same_outcome(got, want, what):
    g, gw, gn = got
    w, ww, wn = want
    if isinstance(w, Exception):
        assert type(g) is type(w) and str(g) == str(w), (what, g, w)
    else:
        assert isinstance(g, np.ndarray), (what, g)
        assert g.dtype == w.dtype and g.shape == w.shape, (what, g.dtype, w.dtype, g.shape, w.shape)
        assert bits_equal(g, w), what
    assert gw == ww, (what, gw, ww)
    assert gn == wn, (what, "random state")


@pytest.mark.parametrize("seed", range(4))
def test_random_calls_against_the_reference(seed):
    ref = _reference()
    rng = np.random.default_rng(2000 + seed)
    declined = 0
    for i in range(60):
        fn, args, kw, unsupported = _random_call(rng)
        what = (fn, [getattr(a, "shape", a) for a in args], getattr(args[0], "dtype", None), kw)
        with cpu_abi_ensemblestats.emulated():
            got = _outcome(_ours(fn), args, kw, seed=i)
        want = _outcome(getattr(ref, fn), args, kw, seed=i)
        if isinstance(got[0], NotImplementedError):
            assert unsupported, (what, got[0])
            declined += 1
            continue
        assert not unsupported or isinstance(want[0], Exception), what
        _same_outcome(got, want, what)
    assert declined < 60


def test_fortran_order_and_views_are_supported():
    """any memory layout: the host makes the members contiguous (NumPy's own values in C order)"""
    ref = _reference()
    rng = np.random.default_rng(5)
    R = rng.gamma(0.8, 2.0, (12, 3, 20, 16))
    view = R[:, -1]
    with cpu_abi_ensemblestats.emulated():
        assert bits_equal(_ours("mean")(view), ref.mean(view))
        assert bits_equal(_ours("excprob")(view, 0.5), ref.excprob(view, 0.5))
        F = np.asfortranarray(view)
        assert bits_equal(_ours("excprob")(F, [0.5, 1.0]), ref.excprob(F, [0.5, 1.0]))
        assert _ours("mean")(F).dtype == np.float64


def test_errstate_is_honoured():
    X = np.full((3, 2, 2), 2e38, np.float32)
    with cpu_abi_ensemblestats.emulated():
        with np.errstate(over="raise"):
            with pytest.raises(FloatingPointError, match="overflow encountered in reduce"):
                _ours("mean")(X)
        with np.errstate(over="ignore"), warnings.catch_warnings():
            warnings.simplefilter("error")
            assert np.isinf(_ours("mean")(X)).all()


@pytest.mark.parametrize("bad", [np.ma.masked_array(np.zeros((2, 3, 3))), np.zeros((2, 3, 3), np.int32)])
def test_unsupported_inputs_raise(bad):
    with cpu_abi_ensemblestats.emulated():
        for fn, args in (("mean", (bad,)), ("excprob", (bad, 0.5)), ("banddepth", (bad,))):
            with pytest.raises(NotImplementedError):
                _ours(fn)(*args)


def test_unsupported_thresholds_raise():
    X = np.zeros((2, 3, 3))
    with cpu_abi_ensemblestats.emulated():
        with pytest.raises(NotImplementedError):
            _ours("excprob")(X, [np.zeros(3)])
        with pytest.raises(NotImplementedError):
            _ours("mean")(X, X_thr=np.zeros((3, 3)))
        with pytest.raises(NotImplementedError):
            _ours("excprob")(X, np.complex128(1))
