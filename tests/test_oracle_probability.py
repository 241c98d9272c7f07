"""CPU: the probability oracle (oracle/probability.py) -- its exact counts against scipy's direct
convolution, its kernel against the reference's, and the whole nowcast against the live reference
and the stored goldens."""
import os

import numpy as np
import pytest
import scipy.signal

from oracle import probability as ora
from probability_cases import CASES, LARGE, build_case, sample_index

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "probability_golden.npz")
BOUND = 1e-6


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.nowcasts.lagrangian_probability")


@pytest.mark.parametrize("shape", [(17, 23), (40, 9), (5, 61), (1, 30), (30, 1), (64, 64)])
def test_counts_equal_direct_convolution(shape):
    rng = np.random.default_rng(shape[0] * 100 + shape[1])
    A = (rng.random(shape) < 0.4).astype(np.int64)
    V = (rng.random(shape) < 0.8).astype(np.int64)
    for s in range(1, 81):
        K = ora.kernel(s)
        for X in (A, V):
            want = scipy.signal.convolve(X, K, mode="same", method="direct")
            assert np.array_equal(ora.counts(X, s), want), (shape, s)


def test_kernel_is_the_references():
    ref = _reference()
    for s in list(range(1, 81)) + [90, 127, 128]:
        assert np.array_equal(ora.kernel(s), ref._get_kernel(s).astype(np.int64)), s


def test_host_run_table_is_the_oracles():
    from pysteps_b200.nowcasts.lagrangian_probability import _kernel_runs
    for s in list(range(1, 300)) + [1000, 4097, 100001]:
        assert np.array_equal(_kernel_runs(s), ora.kernel_runs(s)), s


def _close(got, want, what):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    if (~nan).any():
        d = np.abs(got[~nan] - want[~nan]).max()
        assert d <= BOUND, (what, d)


@pytest.mark.parametrize("name", CASES)
def test_oracle_within_bound_of_the_live_reference(name):
    ref = _reference()
    args, kw = build_case(name)
    want = ref.forecast(*args, **kw)
    got = ora.forecast(*args, **kw)
    assert got.dtype == want.dtype == np.float64 and got.shape == want.shape
    _close(got, want, name)


@pytest.mark.parametrize("name", CASES)
def test_oracle_within_bound_of_the_stored_reference(name):
    g = np.load(GOLDEN)
    args, kw = build_case(name)
    got = ora.forecast(*args, **kw)
    if name in LARGE:
        idx = sample_index(name, got.shape[1:])
        assert np.array_equal(idx, g[name + "/idx"])
        _close(got.reshape(got.shape[0], -1)[:, idx], g[name + "/samples"], name)
        assert np.array_equal(np.isnan(got).reshape(got.shape[0], -1).sum(axis=1), g[name + "/nan_count"])
    else:
        _close(got, g[name + "/out"], name)
    assert g[name + "/deviation"] <= BOUND
