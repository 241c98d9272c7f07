"""CPU: oracle/blending.py against the live reference's linear and salient blending, bit for bit, on
eulerian nowcasts with exact conversions, member maps, NaN/inf fills and the salience edge cases."""
import numpy as np
import pytest

from conftest import bits_equal
from oracle import blending as ora


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.blending.linear_blending")


def make_case(seed, n_now=1, n_nwp=3, dt=np.float64, nwp_dt=None, m=12, n=14, T=6, special=None):
    rng = np.random.default_rng(seed)
    P = np.where(rng.random((m, n)) < 0.4, 0.0, rng.gamma(0.8, 2.0, (m, n))).astype(dt)
    P[rng.random((m, n)) < 0.05] = np.nan
    shape = (n_nwp, T, m, n) if n_nwp > 1 else (T, m, n)
    R = np.where(rng.random(shape) < 0.4, 0.0, rng.gamma(0.8, 2.0, shape)).astype(nwp_dt or dt)
    u = rng.random(shape)
    R[u < 0.05] = np.nan
    if special == "inf":
        R[(u > 0.05) & (u < 0.07)] = np.inf
        R[(u > 0.07) & (u < 0.09)] = -np.inf
    if special == "zero":
        P[:] = 0.0
        R[:] = 0.0
    if special == "negzero":
        P[:] = 0.0
        R[:] = -0.0
    return P, R


CASES = [dict(seed=s, n_nwp=k, dt=dt, special=sp, saliency=sal, fill=fill)
         for s, (k, dt, sp) in enumerate([(1, np.float64, None), (3, np.float64, None), (3, np.float32, None),
                                          (10, np.float64, "inf"), (1, np.float32, "zero"), (3, np.float64, "negzero"),
                                          (1, np.float64, "inf")])
         for sal in (False, True) for fill in (True, False)]


def run_reference(lb, P, R, T, timestep, sal, fill, start=10, end=40, meta=None):
    return lb.forecast(P, meta or {"unit": "mm/h", "transform": None}, np.zeros((2,) + P.shape[-2:]), T, timestep,
                       "eulerian", R, {"unit": "mm/h", "transform": None}, start_blending=start,
                       end_blending=end, fill_nwp=fill, saliency=sal)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_equals_reference(case):
    lb = _reference()
    c = CASES[case]
    P, R = make_case(c["seed"], n_nwp=c["n_nwp"], dt=c["dt"], special=c["special"])
    with np.errstate(all="ignore"):
        want = run_reference(lb, P.copy(), R.copy(), 6, 10, c["saliency"], c["fill"])
        now = np.repeat(P[None], 4, axis=0)
        got = ora.blend(now, R, 6, 10, 10, 40, c["fill"], c["saliency"])
    assert bits_equal(got, want)


def test_member_map_is_consecutive_blocks():
    assert list(ora.member_map(3, 10)) == [0, 0, 0, 1, 1, 1, 2, 2, 2, 2]


def test_dense_rank_equals_rankdata():
    from scipy.stats import rankdata
    rng = np.random.default_rng(0)
    for x in (rng.integers(-3, 4, 500).astype(np.float64), np.array([-0.0, 0.0, 1.0]),
              np.array([np.inf, -np.inf, 5e-324, -5e-324, 0.0]), np.array([1.0, np.nan])):
        assert bits_equal(ora.dense_rank(x), rankdata(x, method="dense").astype(float))
