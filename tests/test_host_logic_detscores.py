"""CPU test of the HOST logic of pysteps_b200.verification's deterministic and spatial scores (argument
checks, axis handling, exceptions and messages, warnings, returned types, dict contents), with the
entry points of csrc/detscores.cu and csrc/fss.cu emulated (tests/cpu_abi_detscores.py).  Compared
with the stored reference outcomes, and with the live reference where it exists on randomised valid
and invalid calls and on dicts passed between the two packages, through *_merge too."""
import os

import numpy as np
import pytest

import cpu_abi_detscores
from detscores_cases import field, golden_calls, our_modules, reference_modules, run_call
from verification_cases import Goldens, matches_golden, same_outcome

GOLDEN = Goldens(os.path.join(os.path.dirname(__file__), "golden", "detscores_golden.npz"))
CALLS = golden_calls()


@pytest.mark.parametrize("i", range(len(CALLS)), ids=[c[0] for c in CALLS])
def test_golden_calls_through_the_host(i):
    key, mod, fn, args, kwargs = CALLS[i]
    with cpu_abi_detscores.emulated():
        out, warned = run_call(our_modules()[mod], fn, args, kwargs)
    problems = matches_golden(GOLDEN, key, out, warned, None)
    assert not problems, (key, problems)


@pytest.fixture(scope="module")
def ref():
    r = reference_modules()
    if r is None:
        pytest.skip("the reference is not present")
    return r


def _thr(rng):
    v = float(rng.choice([0.0, 0.1, 0.5, 1.0, 2.5]))
    kinds = [v, np.float64(v), np.float32(v), int(v), np.array(v)]
    return kinds[int(rng.integers(0, len(kinds)))]


def _dtype(rng):
    return np.int64 if rng.random() < 0.05 else [np.float32, np.float64][int(rng.integers(0, 2))]


def _array(rng, shape):
    dt = _dtype(rng)
    X = field(rng, shape, nans=0.1 * rng.random(), infs=0.05 * rng.random())
    if rng.random() < 0.05:
        X[...] = np.nan
    return np.nan_to_num(X, posinf=9, neginf=-9).astype(dt) if dt == np.int64 else X.astype(dt)


def _axis(rng, nd):
    r = rng.random()
    if r < 0.2:
        return None
    if r < 0.45:
        return int(rng.integers(-2, nd + 1))
    k = int(rng.integers(0, nd + 1))
    return tuple(int(a) for a in rng.integers(-1, nd + (rng.random() < 0.1), size=k))


def _random_call(rng):
    """(module, function, args, kwargs)"""
    which = int(rng.integers(0, 8))
    if which >= 6:  # the continuous scores; no repeated axis (its warnings before NumPy's error are not replayed)
        shape = tuple(int(rng.integers(1 if rng.random() < 0.95 else 0, 6)) for _ in range(int(rng.integers(1, 5))))
        A, B = _array(rng, shape), _array(rng, shape if rng.random() < 0.95 else shape[::-1])
        ax = _axis(rng, len(shape))
        ax = tuple(dict.fromkeys(ax)) if isinstance(ax, tuple) else ax
        cond = [None, None, "single", "double", "x"][int(rng.integers(0, 5))]
        if which == 6:
            scores = [["ME", "rmse", "corr_p", "beta", "beta2", "nmse", "rv", "drmse", "mae"], "MSE", [],
                      ["corr_s"], ""][int(rng.integers(0, 5))]
            return "detcontscores", "det_cont_fct", (A, B, scores, ax, cond, _thr(rng)), {}
        C, D = (A, B) if rng.random() < 0.6 else (_array(rng, A.shape), _array(rng, A.shape))
        return "detcontscores", "det_cont_fct_accum", ((ax, cond, _thr(rng)), (A, B), (C, D)), {}
    if which <= 1:
        shape = tuple(int(rng.integers(1 if rng.random() < 0.95 else 0, 6)) for _ in range(int(rng.integers(1, 5))))
        other = shape if rng.random() < 0.9 else shape[::-1]
        A, B = _array(rng, shape), _array(rng, other)
        ax = _axis(rng, len(shape))
        if which == 0:
            scores = ["", "csi", ["pod", "FAR", "ets"], "SEDI", ["x", None]][int(rng.integers(0, 5))]
            return "detcatscores", "det_cat_fct", (A, B, _thr(rng), scores, ax), {}
        C, D = (A, B) if rng.random() < 0.7 else (_array(rng, shape), _array(rng, shape))
        return "detcatscores", "det_cat_fct_accum", ((_thr(rng), ax), (A, B), (C, D)), {}
    if which <= 3:
        shape = tuple(int(rng.integers(1, 30)) for _ in range(2 if rng.random() < 0.95 else 3))
        A, B = _array(rng, shape), _array(rng, shape if rng.random() < 0.95 else shape[::-1])
        scale = [1, 1.5, 2, 2.5, 3, 7, 40, 0, -1][int(rng.integers(0, 9))]
        if which == 2:
            return "spatialscores", "fss", (A, B, _thr(rng), scale), {}
        thrs = [float(t) for t in rng.choice([0.1, 0.5, 1.0, 2.0], size=int(rng.integers(1, 4)))]
        scales = [int(s) for s in rng.choice([1, 2, 3, 5, 9], size=int(rng.integers(1, 4)))]
        return "spatialscores", "intensity_scale", (A, B, "FSS" if rng.random() < 0.9 else "fss", thrs, scales), {}
    k = int(rng.integers(1, 6))
    shape = tuple(int(rng.integers(1, 20)) for _ in range(2))
    E = _array(rng, (k,) + shape if rng.random() < 0.95 else shape)
    o = _array(rng, shape)
    metric = ["fss", "fss", "CSI", "csi", "HK", "sedi", "RMSE", "rmse", "beta"][int(rng.integers(0, 9))]
    kw = {"thr": _thr(rng)} if metric.lower() not in ("rmse", "beta") else {}
    if metric == "fss":
        kw["scale"] = [1, 2, 3, 5][int(rng.integers(0, 4))]
    if which == 4:
        return "ensscores", "ensemble_skill", (E, o, metric), kw
    return "ensscores", "ensemble_spread", (E, metric), kw


def test_randomised_calls_against_the_reference(ref):
    rng = np.random.default_rng(2025)
    ours = our_modules()
    compared = refused = 0
    for t in range(500):
        mod, fn, args, kwargs = _random_call(rng)
        want = run_call(ref[mod], fn, args, kwargs)
        with cpu_abi_detscores.emulated():
            got = run_call(ours[mod], fn, args, kwargs)
        if isinstance(got[0], NotImplementedError):
            refused += 1
            continue
        compared += 1
        assert same_outcome(got[0], want[0]), (t, fn, args[2:] if fn != "det_cat_fct_accum" else args[0], got[0],
                                               want[0])
        assert got[1] == want[1], (t, fn, got[1], want[1])
    assert compared >= 380 and refused < 120, (compared, refused)


def test_dicts_pass_between_the_reference_and_this_package(ref):
    ours = our_modules()
    rng = np.random.default_rng(8)
    A, B = field(rng, (3, 20, 30), np.float32, nans=0.05), field(rng, (3, 20, 30), nans=0.05)
    plans = (("detcatscores", "det_cat_fct", (1.0, (1, 2)), (A, B)),
             ("detcontscores", "det_cont_fct", ((2,), "single", 0.5), (A, B)),
             ("spatialscores", "fss", (1.0, 5), (A[0], B[0])),
             ("spatialscores", "intensity_scale", ("FSS", [0.5, 1.0], [1, 4]), (A[1], B[1])))
    for mod, name, init_args, data in plans:
        init, accum, merge, compute = (name + s for s in ("_init", "_accum", "_merge", "_compute"))
        for first, second in ((ref, ours), (ours, ref)):
            d = getattr(first[mod], init)(*init_args)
            with cpu_abi_detscores.emulated():
                getattr(ours[mod], accum)(d, *data)
            getattr(ref[mod], accum)(d, *data)
            e = getattr(second[mod], init)(*init_args)
            with cpu_abi_detscores.emulated():
                getattr(ours[mod], accum)(e, *data)
            merged = getattr(second[mod], merge)(d, e)
            got = run_call(second[mod], compute, (merged,), {})
            w = getattr(ref[mod], init)(*init_args)
            for _ in range(3):
                getattr(ref[mod], accum)(w, *data)
            want = run_call(ref[mod], compute, (w,), {})
            assert same_outcome(merged, w), name
            assert same_outcome(got[0], want[0]) and got[1] == want[1], name
