"""CPU: the constant-advection oracle (oracle/constant.py) against NumPy and against the reference's
recorded evaluations (tests/golden/constant_golden.npz, gen_constant_golden.py)."""
import os
import warnings

import numpy as np
import pytest
import scipy.optimize as op
from scipy.ndimage import map_coordinates

from constant_cases import CASES, ORDER_DECIDED, build_case
from oracle import constant as ora

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "constant_golden.npz")


def _same_float(a, b):
    return (np.isnan(a) and np.isnan(b)) or np.float64(a).view(np.int64) == np.float64(b).view(np.int64)


def _np_mean(a):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return float(np.mean(a))


def test_pairwise_mean_matches_numpy_for_every_small_count():
    rng = np.random.default_rng(0)
    for N in range(0, 2001):
        a = rng.standard_normal(N) * 10.0 ** rng.uniform(-4, 4, N)
        assert _same_float(ora.mean(a), _np_mean(a)), N


@pytest.mark.parametrize("N", [255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097, 8191, 8192, 8193, 65535,
                               65536, 65537, 131071, 131073, 999_999, 1_000_000])
def test_pairwise_mean_matches_numpy_at_block_edges(N):
    rng = np.random.default_rng(N)
    a = rng.standard_normal(N) * 10.0 ** rng.uniform(-4, 4, N) + 3.0
    assert _same_float(ora.mean(a), _np_mean(a))
    # the mean numpy's np.cov takes: one row of a (2, N) array
    X = np.vstack([a, a[::-1]])
    assert _same_float(ora.mean(a[::-1]), float(X.mean(axis=1)[1]))


@pytest.mark.parametrize("N,expect", [(3, 0.0), (10, np.nan), (1000, 0.0)])
def test_constant_values_against_a_ramp(N, expect):
    """0.1 repeated: numpy's mean is exactly 0.1 only for some counts, and corrcoef follows it"""
    a, b = np.full(N, 0.1), np.arange(N, dtype=np.float64)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        want = np.corrcoef(a, b)[0, 1]
    f, flags = ora.tail(*ora.centred_sums(a, b, ora.mean(a), ora.mean(b)), N)
    assert _same_float(-f, want) if not np.isnan(expect) else np.isnan(f)
    invalid = [str(x.message) for x in w].count("invalid value encountered in divide")
    assert invalid == (2 if np.isnan(expect) else 0)
    assert flags == (ora.ROW_INVALID | ora.COL_INVALID if np.isnan(expect) else 0)


def _reference_objective(prev, nxt, v):
    """constant.py:41-49 with the frames given"""
    m, n = nxt.shape
    X, Y = np.meshgrid(np.arange(n), np.arange(m))
    R_w = map_coordinates(prev, [Y + v[1], X + v[0]], mode="constant", cval=np.nan, order=0, prefilter=False)
    mask = np.logical_and(np.isfinite(nxt), np.isfinite(R_w))
    return -np.corrcoef(nxt[mask], R_w[mask])[0, 1], int(mask.sum())


def test_taps_and_counts_match_map_coordinates_near_half_integers():
    rng = np.random.default_rng(3)
    comps = [0.5, 0.49999999999999994, -0.5, 2.5, -0.49999999999999994, 1.5000000000000002, -3.5, 0.0]
    for _ in range(60):
        m, n = (int(k) for k in rng.integers(1, 300, 2))
        R = rng.standard_normal((2, m, n))
        R[rng.random((2, m, n)) < 0.05] = np.nan
        v = rng.choice(comps, 2)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want, count = _reference_objective(R[0], R[1], v)
            f, N, _ = ora.evaluate(R[0], R[1], v[0], v[1])
        assert N == count
        assert (np.isnan(f) and np.isnan(want)) or abs(f - want) <= 1e-12


def _close(a, b):
    return (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-12


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_every_recorded_evaluation(name):
    g = np.load(GOLDEN)
    R = np.ma.getdata(build_case(name))
    for k, (v, want) in enumerate(zip(g[name + "/v"], g[name + "/f"])):
        got = ora.evaluate(R[-2], R[-1], v[0], v[1])[0]
        assert _close(got, want), (k, v, got, want)


def _oracle_path(R):
    seen = []
    prev, nxt = np.ma.getdata(R)[-2], np.ma.getdata(R)[-1]

    def f(v):
        val = ora.evaluate(prev, nxt, v[0], v[1])[0]
        seen.append((np.array(v), val))
        return val

    options = {"initial_simplex": (np.array([(0, 1), (1, 0), (1, 1)]))}
    return op.minimize(f, (1, 1), method="Nelder-Mead", options=options), seen


@pytest.mark.parametrize("name", [c for c in CASES if c not in ORDER_DECIDED])
def test_oracle_through_scipy_gives_the_reference_result(name):
    """Nelder-Mead on the oracle objective visits exactly the reference's points and ends at the
    reference's result.x"""
    g = np.load(GOLDEN)
    res, seen = _oracle_path(build_case(name))
    gv = g[name + "/v"]
    assert len(seen) == len(gv)
    assert all(np.array_equal(v, gv[k]) for k, (v, _) in enumerate(seen))
    assert np.array_equal(res.x, g[name + "/x"])


@pytest.mark.parametrize("name", sorted(ORDER_DECIDED))
def test_order_decided_cases_part_at_the_named_tie(name):
    """The path leaves the reference's right after the named pair of evaluations: different points,
    reference f within 1e-12 of each other, ordered the other way by the oracle's summation order.
    Both runs end on the same plateau of f."""
    g = np.load(GOLDEN)
    R = build_case(name)
    res, seen = _oracle_path(R)
    gv, gf = g[name + "/v"], g[name + "/f"]
    i, j = ORDER_DECIDED[name]
    k = next(k for k, (v, _) in enumerate(seen) if k >= len(gv) or not np.array_equal(v, gv[k]))
    assert j < k <= j + 2, k
    assert not np.array_equal(gv[i], gv[j]) and abs(gf[i] - gf[j]) <= 1e-12
    oi, oj = seen[i][1], seen[j][1]
    assert np.sign(gf[i] - gf[j]) != np.sign(oi - oj)
    data = np.ma.getdata(R)
    at_ours = ora.evaluate(data[-2], data[-1], *res.x)[0]
    at_ref = ora.evaluate(data[-2], data[-1], *g[name + "/x"])[0]
    assert abs(at_ours - at_ref) <= 1e-12 and abs(at_ours + 1.0) <= 1e-12
