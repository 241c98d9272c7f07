"""CPU test of the oracle of the deterministic and spatial verification scores (oracle/detscores.py):
the contingency counts and the FSS sums bit for bit against the live reference's accumulators, the
running-sum filter against scipy.ndimage.uniform_filter, and the spread as the reference's pair loop."""
import itertools
import warnings

import numpy as np
import pytest
from scipy.ndimage import uniform_filter

from detscores_cases import field, reference_modules
from oracle import detscores as ora


@pytest.fixture(scope="module")
def ref():
    r = reference_modules()
    if r is None:
        pytest.skip("the reference is not present")
    return r


def test_uniform_filter_matches_scipy():
    rng = np.random.default_rng(41)
    for (m, n), p in itertools.product([(64, 80), (7, 5), (200, 131), (1, 9), (33, 1)], (0.05, 0.5, 0.9)):
        I = (rng.random((m, n)) < p).astype(float)
        for s in (2, 3, 4, 5, 8, 11, 16, 25, 40, 81, 301):
            want = uniform_filter(I, size=s, mode="constant", cval=0.0)
            assert ora.uniform_filter(I, s).tobytes() == want.tobytes(), (m, n, p, s)
        assert uniform_filter(I, size=2.5, mode="constant").tobytes() == ora.uniform_filter(I, 2).tobytes()


@pytest.mark.parametrize("shape", [(50,), (7, 9), (4, 6, 5), (3, 1, 4, 5), (2, 3, 1, 6)])
def test_contab_matches_the_reference(ref, shape):
    rng = np.random.default_rng(42)
    A = field(rng, shape, nans=0.1, infs=0.1)
    B = field(rng, shape, np.float32, nans=0.1, infs=0.1)
    nd = len(shape)
    for r in range(1, nd + 1):
        for axis in itertools.combinations(range(nd), r):
            for thr in (0.5, np.float64(0.5), np.float32(1.1), np.array(2.0)):
                d = ref["detcatscores"].det_cat_fct_init(thr, axis)
                ref["detcatscores"].det_cat_fct_accum(d, A, B)
                got = ora.contab(A, B, thr, axis)
                for key, g in zip(("hits", "false_alarms", "misses", "correct_negatives"), got):
                    assert np.array_equal(d[key], g), (axis, thr, key)


@pytest.mark.parametrize("scale", [1, 1.5, 2, 3, 16, 60])
@pytest.mark.parametrize("dtypes", [(np.float64, np.float64), (np.float32, np.float64), (np.float32, np.float32)])
def test_fss_sums_match_the_reference(ref, scale, dtypes):
    rng = np.random.default_rng(43)
    X = field(rng, (41, 37), dtypes[0], nans=0.05, infs=0.05)
    Y = field(rng, (41, 37), dtypes[1], nans=0.05)
    for thr in (1.0, np.float32(0.3), 1e8):
        d = ref["spatialscores"].fss_init(thr, scale)
        ref["spatialscores"].fss_accum(d, X * 1e8 if thr == 1e8 else X, Y)
        got = ora.fss_sums(X * 1e8 if thr == 1e8 else X, Y, thr, scale)
        for key, g in zip(("sum_obs_sq", "sum_fct_obs", "sum_fct_sq"), got):
            assert np.float64(d[key]).tobytes() == np.float64(g).tobytes(), (thr, key)


def test_spread_matches_the_reference(ref):
    rng = np.random.default_rng(44)
    E = field(rng, (5, 30, 22), nans=0.05)
    want = ref["ensscores"].ensemble_spread(E, "fss", thr=1.0, scale=4)
    assert np.float64(want).tobytes() == np.mean(ora.spread_fss(E, 1.0, 4)).tobytes()


@pytest.mark.parametrize("dtypes", [(np.float64, np.float64), (np.float32, np.float64), (np.float32, np.float32)])
def test_moments_match_the_reference(ref, dtypes):
    """the oracle's nine means, divided as NumPy divides, through the reference's own updates equal the
    reference's dict"""
    import importlib
    rc = importlib.import_module("pysteps.verification.detcontscores")
    rng = np.random.default_rng(45)
    A = field(rng, (4, 1, 9, 13), dtypes[0], nans=0.05, infs=0.05)
    B = field(rng, (4, 1, 9, 13), dtypes[1], nans=0.05, infs=0.02)
    compared = 0
    for axis in [(0,), (2, 3), (0, 2), (0, 1, 2, 3), (1,), (1, 2, 3)]:
        for cond in (None, "single", "double"):
            got = rc.det_cont_fct_init(axis, cond, 0.5)
            with np.errstate(all="ignore"), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                try:
                    rc.det_cont_fct_accum(got, A, B)
                except IndexError:  # the reference's squeeze of the means fails for a kept unit axis
                    continue
                tot, cnt, n = ora.cont_sums(A, B, axis, cond, 0.5)
                m = [(t.astype(np.float64) / c).astype(t.dtype) for t, c in zip(tot, cnt)]
                mo, mp = np.asarray(m[0]).squeeze(), np.asarray(m[1]).squeeze()
                want = rc.det_cont_fct_init(axis, cond, 0.5)
                for key in ("cov", "vobs", "vpred", "mobs", "mpred", "me", "mse", "mss", "mae", "n"):
                    want[key] = np.zeros(n.shape)
                rc._parallel_var(want["mobs"], want["n"], want["vobs"], mo, n, m[7])
                rc._parallel_var(want["mpred"], want["n"], want["vpred"], mp, n, m[8])
                rc._parallel_cov(want["cov"], want["mobs"], want["mpred"], want["n"], m[6], mo, mp, n)
                for key, v in zip(("mobs", "mpred", "me", "mse", "mss", "mae"), (mo, mp) + tuple(m[2:6])):
                    rc._parallel_mean(want[key], want["n"], v, n)
                want["n"] += n
            for key in want:
                assert np.asarray(got[key]).tobytes() == np.asarray(want[key]).tobytes(), (axis, cond, key)
            compared += 1
    assert compared >= 9

