"""CPU: the ensemble-statistics oracle (oracle/ensemblestats.py) against the reference's stored outputs
(tests/golden/ensemblestats_golden.npz) and, where it is importable, against the live reference,
bit for bit."""
import os
import warnings

import numpy as np
import pytest

from conftest import assert_bits_equal
from ensemblestats_cases import CASES, LARGE, build_case, rain, nonfinite, sample_index, seed_of
from oracle import ensemblestats as ora

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ensemblestats_golden.npz")


def _quiet(fn, *args, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*args, **kw)


def oracle_call(name):
    """the oracle's output of a golden case (banddepth with the tie-breaks of the case's seed)"""
    fn, args, kw = build_case(name)
    if fn != "banddepth":
        return _quiet(getattr(ora, fn), *args, **kw)
    X = args[0]
    thr = kw.get("thr")
    if thr is None:
        thr = _quiet(np.nanmin, X)
    mask, _ = ora.band_mask(X, thr)
    np.random.seed(seed_of(name))
    b = np.random.random((X.shape[0], int(mask.sum())))
    return _quiet(ora.banddepth, X, b, thr=thr, norm=kw.get("norm", False))


def check_golden(name, got):
    """got (the full output of case `name`) against the stored reference output, bit for bit"""
    g = np.load(GOLDEN)
    if name in LARGE:
        planes = got.reshape(-1, got.shape[-2] * got.shape[-1])
        idx = sample_index(name, planes.shape[1])
        assert np.array_equal(g[name + "/idx"], idx)
        assert_bits_equal(planes[:, idx], g[name + "/samples"], name)
        assert np.array_equal(np.isnan(planes).sum(axis=1), g[name + "/nan_count"]), name
    else:
        assert_bits_equal(got, g[name + "/out"], name)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_golden(name):
    check_golden(name, oracle_call(name))


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.postprocessing.ensemblestats")


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_the_live_reference(seed):
    ref = _reference()
    rng = np.random.default_rng(100 + seed)
    dt = (np.float32, np.float64)[seed % 2]
    k = int(rng.choice([1, 2, 5, 24]))
    X = rain(k, (int(rng.integers(1, 40)), int(rng.integers(1, 40))), seed, dt)
    if seed >= 3:
        X = nonfinite(X, seed, frac=0.1, all_nan_pixels=1)
    thr = [float(v) for v in rng.random(3) * 2]
    for ignore_nan in (False, True):
        assert_bits_equal(_quiet(ora.mean, X, ignore_nan), _quiet(ref.mean, X, ignore_nan))
        assert_bits_equal(_quiet(ora.mean, X, ignore_nan, thr[0]), _quiet(ref.mean, X, ignore_nan, thr[0]))
        assert_bits_equal(_quiet(ora.excprob, X, thr, ignore_nan), _quiet(ref.excprob, X, thr, ignore_nan))
        assert_bits_equal(_quiet(ora.excprob, X, thr[1], ignore_nan), _quiet(ref.excprob, X, thr[1], ignore_nan))
    for kw in ({}, {"thr": thr[2]}, {"norm": True}):
        t = kw.get("thr")
        if t is None:
            t = _quiet(np.nanmin, X)
        mask, _ = ora.band_mask(X, t)
        np.random.seed(seed)
        b = np.random.random((k, int(mask.sum())))
        np.random.seed(seed)
        assert_bits_equal(_quiet(ora.banddepth, X, b, **kw), _quiet(ref.banddepth, X, **kw))


def test_rank_identity_on_ties():
    """1 + #{j : (X_j, b_j) < (X_i, b_i)}, lower index first on a full tie, is lexsort's rank"""
    rng = np.random.default_rng(7)
    X = rng.integers(0, 3, (9, 500)).astype(np.float64)
    X[X == 1] = -0.0 * (rng.random(int((X == 1).sum())) < 0.5)  # -0.0 and 0.0 compare equal
    b = rng.integers(0, 4, X.shape) / 4.0  # full ties of both keys
    mask = np.ones(500, dtype=bool)
    rank = np.lexsort((b, X), axis=0).argsort(axis=0) + 1
    assert np.array_equal(ora.band_match(X, mask, b), ((9 - rank) * (rank - 1)).sum(axis=1))
