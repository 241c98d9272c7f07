"""The verification scores on the device (pysteps_b200.verification) against the oracle
(oracle/verification.py) and the live reference where it is present: accumulator dicts bit for bit,
the warnings of the compute steps, the random state after the rank histogram, NumPy and CUDA-tensor
input, float32 and float64, repeated and accumulated calls, and the calls that must be refused
before any launch."""
import warnings
from unittest import mock

import numpy as np
import pytest
import torch

from oracle import verification as ora
import os

from verification_cases import (Goldens, ensemble_cases, flip_zeros, golden_calls, matches_golden, prob_cases, rain,
                                reference, run_call)

pytestmark = pytest.mark.gpu
ENS = ensemble_cases()
PROB = prob_cases()
GOLDEN = Goldens(os.path.join(os.path.dirname(__file__), "golden", "verification_golden.npz"))
CALLS = golden_calls()


@pytest.mark.parametrize("i", range(len(CALLS)), ids=[c[0] for c in CALLS])
def test_golden_calls(i):
    """every stored reference outcome: types, values bit for bit, warnings and the next random draw"""
    key, mod, fn, args, seed = CALLS[i]
    ps, es = _ours()
    out, warned, nxt = run_call(ps if mod == "probscores" else es, fn, args, seed)
    problems = matches_golden(GOLDEN, key, out, warned, nxt)
    assert not problems, (key, problems)


@pytest.mark.parametrize("name", [n for n in sorted(ENS) if "zeros" in n or n.startswith("k")])
def test_crps_does_not_depend_on_the_sign_of_zeros(name):
    ps, _ = _ours()
    X_f, X_o, _ = ENS[name]
    a, b = ps.CRPS_init(), ps.CRPS_init()
    ps.CRPS_accum(a, X_f, X_o)
    ps.CRPS_accum(b, flip_zeros(X_f), X_o)
    assert a["CRPS_sum"].tobytes() == b["CRPS_sum"].tobytes() and a["n"] == b["n"]


def _ours():
    from pysteps_b200.verification import ensscores, probscores
    return probscores, ensscores


def _outcome(fn, *args):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            out = fn(*args)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            out = e
    return out, [f"{x.category.__name__}: {x.message}" for x in w]


def _same(a, b):
    if isinstance(a, Exception) or isinstance(b, Exception):
        return type(a) is type(b) and str(a) == str(b)
    if isinstance(a, (tuple, list)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return type(a) is type(b) and a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return type(a) is type(b) and (a == b or (a != a and b != b)) and np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _crps_check(X_f, X_o, as_tensor=False, want=None):
    ps, _ = _ours()
    d = ps.CRPS_init()
    f, o = (torch.from_numpy(X_f).cuda(), torch.from_numpy(X_o).cuda()) if as_tensor else (X_f, X_o)
    ps.CRPS_accum(d, f, o)
    s, n = want or ora.crps(X_f, X_o)
    assert type(d["CRPS_sum"]) is np.float64 and type(d["n"]) is float
    assert d["CRPS_sum"].tobytes() == np.float64(0.0 + s).tobytes() and d["n"] == n
    return d


def _rankhist_check(X_f, X_o, X_min, as_tensor=False):
    _, es = _ours()
    f, o = (torch.from_numpy(X_f).cuda(), torch.from_numpy(X_o).cuda()) if as_tensor else (X_f, X_o)
    np.random.seed(7)
    h = es.rankhist_init(X_f.shape[0], X_min)
    es.rankhist_accum(h, f, o)
    nxt = np.random.random()
    counts, pairs = ora.rankhist(X_f, X_o, X_min)
    np.random.seed(7)
    u = np.random.uniform(size=len(pairs)) if len(pairs) else np.zeros(0)
    assert np.random.random() == nxt, "the random state after rankhist differs"
    want = ora.rankhist(X_f, X_o, X_min, u)
    assert h["n"].dtype == np.int64 and np.array_equal(h["n"], want)


@pytest.mark.parametrize("name", sorted(ENS))
def test_crps_and_rankhist_cases(name):
    X_f, X_o, X_min = ENS[name]
    _crps_check(X_f, X_o)
    for xm in (None, X_min):
        _rankhist_check(X_f, X_o, xm)


@pytest.mark.parametrize("name", sorted(ENS))
def test_wrappers_match_the_reference(name):
    ref = reference()
    if ref is None:
        pytest.skip("the reference is not present")
    X_f, X_o, X_min = ENS[name]
    ours = _ours()
    for mod, fn, args in ((0, "CRPS", (X_f, X_o)), (1, "rankhist", (X_f, X_o, X_min)),
                          (1, "rankhist", (X_f, X_o, X_min, False))):
        np.random.seed(3)
        want = _outcome(getattr(ref[mod], fn), *args) + (np.random.random(),)
        np.random.seed(3)
        got = _outcome(getattr(ours[mod], fn), *args) + (np.random.random(),)
        assert _same(got[0], want[0]) and got[1] == want[1] and got[2] == want[2], (fn, got, want)


@pytest.mark.parametrize("name", sorted(PROB))
def test_reldiag_and_roc_cases(name):
    ref = reference()
    P, O, X_min, nb = PROB[name]
    ps, _ = _ours()
    for min_count in (0, 10, 11, 100):
        r = ps.reldiag_init(X_min, nb, min_count)
        ps.reldiag_accum(r, P, O)
        count, above, sums = ora.reldiag(P, O, X_min, r["bin_edges"])
        keep = count >= min_count
        assert np.array_equal(r["num_idx"], np.where(keep, count, 0))
        assert np.array_equal(r["sample_size"], np.where(keep, count, 0))
        assert np.array_equal(r["Y_sum"], np.where(keep, above, 0))
        assert r["X_sum"].tobytes() == np.where(keep, sums.astype(np.float64), 0.0).tobytes()
        if ref is not None:
            want = _outcome(ref[0].reldiag, P, O, X_min, nb, min_count)
            got = _outcome(ps.reldiag, P, O, X_min, nb, min_count)
            assert _same(got[0], want[0]) and got[1] == want[1], (got, want)
    roc = ps.ROC_curve_init(X_min, nb)
    ps.ROC_curve_accum(roc, P, O)
    for key, v in zip(("hits", "misses", "false_alarms", "corr_neg"), ora.roc(P, O, X_min, roc["prob_thrs"])):
        assert roc[key].dtype == np.int64 and np.array_equal(roc[key], v), key
    if ref is not None:
        for area in (False, True):
            want = _outcome(ref[0].ROC_curve, P, O, X_min, nb, area)
            got = _outcome(ps.ROC_curve, P, O, X_min, nb, area)
            assert _same(got[0], want[0]) and got[1] == want[1], (got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_large_ensemble_numpy_and_tensor(dtype):
    rng = np.random.default_rng(21)
    X_f = rain(rng, (24, 2048, 2048), dtype, zeros=0.6, nans=1e-4)
    X_o = rain(rng, (2048, 2048), dtype, zeros=0.6)
    want = ora.crps(X_f, X_o)
    for as_tensor in (False, True, True):
        _crps_check(X_f, X_o, as_tensor, want)
        _rankhist_check(X_f, X_o, 0.1, as_tensor)
    P = (X_f >= 1.0).mean(axis=0).astype(dtype)
    ps, _ = _ours()
    for as_tensor in (False, True):
        p, o = (torch.from_numpy(P).cuda(), torch.from_numpy(X_o).cuda()) if as_tensor else (P, X_o)
        r = ps.reldiag_init(1.0, 10, 10)
        ps.reldiag_accum(r, p, o)
        count, above, sums = ora.reldiag(P, X_o, 1.0, r["bin_edges"])
        keep = count >= 10
        assert r["X_sum"].tobytes() == np.where(keep, sums.astype(np.float64), 0.0).tobytes()
        assert np.array_equal(r["Y_sum"], np.where(keep, above, 0))
        roc = ps.ROC_curve_init(1.0, 10)
        ps.ROC_curve_accum(roc, p, o)
        for key, v in zip(("hits", "misses", "false_alarms", "corr_neg"), ora.roc(P, X_o, 1.0, roc["prob_thrs"])):
            assert np.array_equal(roc[key], v), key


def test_k300_ensemble():
    rng = np.random.default_rng(22)
    X_f = rain(rng, (300, 64, 64), np.float32, zeros=0.5)
    X_o = rain(rng, (64, 64), np.float32, zeros=0.5)
    _crps_check(X_f, X_o)
    _crps_check(X_f, X_o, True)
    _rankhist_check(X_f, X_o, 0.1)


def test_twelve_lead_times_accumulate():
    rng = np.random.default_rng(23)
    ps, es = _ours()
    crps, total, n = ps.CRPS_init(), np.float64(0.0), 0
    np.random.seed(9)
    h = es.rankhist_init(12, 0.1)
    draws = []
    for t in range(12):
        X_f = rain(rng, (12, 96, 80), np.float32, zeros=0.6, nans=0.01)
        X_o = rain(rng, (96, 80), np.float32, zeros=0.6)
        ps.CRPS_accum(crps, X_f, X_o)
        s, c = ora.crps(X_f, X_o)
        total, n = total + s, n + c
        draws.append((X_f, X_o))
        es.rankhist_accum(h, X_f, X_o)
    assert crps["CRPS_sum"].tobytes() == (0.0 + total).tobytes() and crps["n"] == n
    nxt = np.random.random()
    np.random.seed(9)
    want = np.zeros(13, np.int64)
    for X_f, X_o in draws:
        pairs = ora.rankhist(X_f, X_o, 0.1)[1]
        want += ora.rankhist(X_f, X_o, 0.1, np.random.uniform(size=len(pairs)) if len(pairs) else np.zeros(0))
    assert np.random.random() == nxt and np.array_equal(h["n"], want)
    assert ps.CRPS_compute(crps) == (1.0 * (0.0 + total)) / float(n)


def test_mixed_accumulation_with_the_reference():
    ref = reference()
    if ref is None:
        pytest.skip("the reference is not present")
    ps, es = _ours()
    rps, res = ref
    X_f, X_o, X_min = ENS["f32_f64_half"]
    P, O, Pmin, nb = PROB["n10"]
    for init, accum, compute, args, data in (
            ("CRPS_init", "CRPS_accum", "CRPS_compute", (), (X_f, X_o)),
            ("reldiag_init", "reldiag_accum", "reldiag_compute", (Pmin, nb, 5), (P, O)),
            ("ROC_curve_init", "ROC_curve_accum", "ROC_curve_compute", (Pmin, nb), (P, O))):
        for make, finish in ((rps, ps), (ps, rps)):
            d = getattr(make, init)(*args)
            getattr(ps if make is rps else rps, accum)(d, *data)
            getattr(ps, accum)(d, *data)
            want = getattr(rps, init)(*args)
            getattr(rps, accum)(want, *data)
            getattr(rps, accum)(want, *data)
            assert _same(d, want), init
            assert _same(_outcome(getattr(finish, compute), d), _outcome(getattr(rps, compute), want))
    for make in (res, es):
        np.random.seed(4)
        d = make.rankhist_init(X_f.shape[0], X_min)
        es.rankhist_accum(d, X_f, X_o)
        res.rankhist_accum(d, X_f, X_o)
        np.random.seed(4)
        want = res.rankhist_init(X_f.shape[0], X_min)
        res.rankhist_accum(want, X_f, X_o)
        res.rankhist_accum(want, X_f, X_o)
        assert _same(d, want) and _same(res.rankhist_compute(d), es.rankhist_compute(want))


def test_refused_before_any_launch():
    from pysteps_b200 import _lib
    ps, es = _ours()
    X = np.zeros((3, 4, 5))
    refused = [
        (ps.CRPS, (X.astype(np.int64), X[0])),
        (ps.CRPS, (np.ma.masked_array(X), X[0])),
        (ps.CRPS, (torch.zeros(3, 4, 5, dtype=torch.float64), X[0])),
        (ps.CRPS, (np.zeros((513, 2, 2)), np.zeros((2, 2)))),
        (es.rankhist, (np.zeros((513, 2, 2)), np.zeros((2, 2)))),
        (ps.reldiag, (X[0], X[0], 0.5, 2049)),
        (ps.ROC_curve, (X[0], X[0], 0.5, 2049)),
        (ps.reldiag, (X[0], X[0], None)),
        (es.rankhist, (np.broadcast_to(np.float32(0), (1, 1 << 31)), np.broadcast_to(np.float32(0), (1 << 31,)))),
    ]
    with mock.patch.object(_lib, "call", side_effect=AssertionError("launched")):
        for fn, args in refused:
            with pytest.raises(NotImplementedError):
                fn(*args)


CATEGORICAL = ("acc", "bias", "csi", "f1", "fa", "far", "gss", "hk", "hss", "mcc", "pod", "sedi")
CONTINUOUS = ("beta", "beta1", "beta2", "corr_p", "corr_s", "drmse", "mae", "mse", "me", "nmse", "rmse", "rv",
              "scatter")


def test_get_method():
    from pysteps_b200 import verification
    ps, es = _ours()
    built = {("crps", "probabilistic"): ps.CRPS, ("reldiag", "probabilistic"): ps.reldiag,
             ("roc", "probabilistic"): ps.ROC_curve, ("rankhist", "ensemble"): es.rankhist}
    not_built = [(n, "deterministic") for n in CATEGORICAL + CONTINUOUS + ("binary_mse", "fss", "sal")] \
        + [("ens_skill", "ensemble"), ("ens_spread", "ensemble")]
    for name, kind in list(built) + not_built:
        for n, t in ((name, kind), (name.upper(), kind.upper()), (name.capitalize(), kind.title())):
            if (name, kind) in built:
                assert verification.get_method(n, t) is built[(name, kind)], (n, t)
            else:
                with pytest.raises(NotImplementedError, match="pysteps.verification"):
                    verification.get_method(n, t)
    with pytest.raises(NotImplementedError):
        verification.get_method("mse")  # type defaults to "deterministic"
    # names known under another type, unknown names and None, for every type
    for kind in ("deterministic", "ensemble", "probabilistic"):
        known = {n for n, t in list(built) + not_built if t == kind}
        for name in ("crps", "rankhist", "ens_skill", "mse", "nope", None):
            if name in known:
                continue
            with pytest.raises(ValueError, match=f"^unknown {kind} method {name or 'none'}$"):
                verification.get_method(name, kind)
    for name in ("crps", "x", None):
        for kind in ("nope", None, "PROBABILISTIC "):
            with pytest.raises(ValueError, match=f"^unknown type {name or 'none'}$"):
                verification.get_method(name, kind)
