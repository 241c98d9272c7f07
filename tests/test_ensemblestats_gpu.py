"""GPU: the ensemble statistics (csrc/ensemblestats.cu behind postprocessing/ensemblestats.py) against
the oracle (oracle/ensemblestats.py) and the reference's stored outputs, warnings and random draws
(tests/golden/ensemblestats_golden.npz), bit for bit."""
import os
import warnings

import numpy as np
import pytest

from conftest import assert_bits_equal
from ensemblestats_cases import CASES, build_case, nonfinite, rain, seed_of
from oracle import ensemblestats as ora
from test_oracle_ensemblestats import check_golden, oracle_call

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ensemblestats_golden.npz")


def _fn(name):
    import pysteps_b200
    return pysteps_b200.postprocessing.get_method(name, "ensemblestats")


def _recorded(fn, *args, **kw):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = fn(*args, **kw)
    return out, [f"{x.category.__name__}: {x.message}" for x in w]


def _quiet(fn, *args, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*args, **kw)


@pytest.mark.parametrize("name", CASES)
def test_golden_case(name):
    fn, args, kw = build_case(name)
    if fn == "banddepth":
        np.random.seed(seed_of(name))
    got, warned = _recorded(_fn(fn), *args, **kw)
    g = np.load(GOLDEN)
    if fn == "banddepth":
        assert np.random.random() == g[name + "/next"], "the random state after the call differs"
    assert_bits_equal(got, oracle_call(name), name)
    check_golden(name, got)
    assert warned == list(g[name + "/warnings"]), name


def _ensemble_2048(dtype):
    return nonfinite(rain(24, (2048, 2048), 61, dtype), 61, frac=0.01, all_nan_pixels=50)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mean_and_excprob_at_24x2048(dtype):
    import torch
    X = _ensemble_2048(dtype)
    d = torch.from_numpy(X).cuda()
    thr4 = [0.1, 0.5, 1.0, 5.0]
    calls = [("mean", (), {}), ("mean", (), {"ignore_nan": True}), ("mean", (), {"X_thr": 0.1}),
             ("excprob", (0.5,), {}), ("excprob", (thr4,), {}), ("excprob", (thr4,), {"ignore_nan": True})]
    for fn, args, kw in calls:
        got = _quiet(_fn(fn), X, *args, **kw)
        assert_bits_equal(got, _quiet(getattr(ora, fn), X, *args, **kw), (fn, kw))
        dev = _quiet(_fn(fn), d, *args, **kw)
        assert dev.is_cuda
        assert_bits_equal(dev.cpu().numpy(), got, ("CUDA-tensor call", fn, kw))
        assert_bits_equal(_quiet(_fn(fn), d, *args, **kw).cpu().numpy(), got, ("repeated call", fn, kw))


def test_banddepth_at_24x2048():
    import torch
    X = rain(24, (2048, 2048), 62, np.float32, zeros=0.6)
    X[:, :8, :8] = np.nan
    np.random.seed(5)
    got = _fn("banddepth")(X)
    after = np.random.random()
    thr = np.nanmin(X)
    mask, _ = ora.band_mask(X, thr)
    np.random.seed(5)
    b = np.random.random((24, int(mask.sum())))
    assert np.random.random() == after
    assert_bits_equal(got, ora.banddepth(X, b), "banddepth 24 x 2048^2")
    np.random.seed(5)
    dev = _fn("banddepth")(torch.from_numpy(X).cuda())
    assert dev.is_cuda and dev.dtype == torch.float64
    assert_bits_equal(dev.cpu().numpy(), got, "CUDA-tensor banddepth")


def test_views_and_fortran_order():
    """a view whose member axis is outermost is bit-identical to NumPy; Fortran order (pairwise
    summation in NumPy) is within the rounding bound of DESIGN.md section 4; counts are exact"""
    rng = np.random.default_rng(63)
    R = rng.gamma(0.8, 2.0, (24, 3, 300, 200)).astype(np.float32)
    view = R[:, -1]
    assert_bits_equal(_fn("mean")(view), np.mean(view, axis=0), "R[:, -1]")
    F = np.asfortranarray(view)
    got, want = _fn("mean")(F), np.mean(F, axis=0)
    eps = np.finfo(np.float32).eps
    bound = 2 * eps * np.abs(F).sum(axis=0, dtype=np.float64)
    assert (np.abs(got.astype(np.float64) - want) <= bound).all()
    got, want = _fn("mean")(F, ignore_nan=True), np.nanmean(F, axis=0)
    assert (np.abs(got.astype(np.float64) - want) <= bound).all()
    assert_bits_equal(_fn("excprob")(F, [0.5, 2.0]), ora.excprob(view, [0.5, 2.0]), "Fortran excprob")


def test_large_k_loops_over_members():
    X = rain(300, (40, 50), 64)
    assert_bits_equal(_fn("mean")(X), ora.mean(X), "k = 300 mean")
    assert_bits_equal(_fn("excprob")(X, [0.5, 1.0]), ora.excprob(X, [0.5, 1.0]), "k = 300 excprob")
    np.random.seed(9)
    got = _fn("banddepth")(X, thr=0.5)
    mask, _ = ora.band_mask(X, 0.5)
    np.random.seed(9)
    b = np.random.random((300, int(mask.sum())))
    assert_bits_equal(got, ora.banddepth(X, b, thr=0.5), "k = 300 banddepth")
