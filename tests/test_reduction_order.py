"""CPU test of NumPy's summation order as the deterministic scores restate it: the host's launch plan
(pysteps_b200.verification._reduction.plan) and the oracle's reduce_sum against np.sum bit for bit, for
every axis subset of shapes up to 4-D with size-1 axes and short trailing runs, in float32 and float64,
and the oracle's nine np.nanmean sums of det_cont_fct_accum against NumPy's own."""
import itertools

import numpy as np
import pytest

from oracle import detscores as ora
from oracle.verification import pairwise
from pysteps_b200.verification import _reduction

SHAPES = [(1000,), (9,), (5000, 3), (3, 5000), (130, 1), (1, 130), (7, 1, 300), (1, 9, 130), (40, 7, 300),
          (300, 7, 40), (1, 1, 17), (17, 1, 1), (2, 3, 4, 200), (5, 1, 9, 1), (3, 1000, 1, 9), (4, 3, 2, 129)]


def _data(rng, shape, dtype):
    return (rng.standard_normal(shape) * 10 ** rng.uniform(-3, 6, shape)).astype(dtype)


def _planned_sum(a, axis):
    """np.sum(a, axis) evaluated in the order of the host's plan"""
    (ks, kst), (os_, ost), L = _reduction.plan(a.shape, axis)
    flat = a.reshape(-1)

    def offsets(sizes, strides):
        off = np.zeros(1, np.int64)
        for n, s in zip(sizes, strides):
            off = (off[:, None] + np.arange(n) * s).reshape(-1)
        return off

    base = offsets(ks, kst)
    out = np.zeros(len(base), a.dtype)
    for o in offsets(os_, ost):
        runs = flat[(base + o)[:, None] + np.arange(L)[None, :]]
        out = out + pairwise(runs)
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_plan_and_oracle_match_np_sum(shape, dtype):
    rng = np.random.default_rng(len(shape) * 1000 + shape[-1])
    a = _data(rng, shape, dtype)
    for r in range(1, len(shape) + 1):
        for axis in itertools.combinations(range(len(shape)), r):
            want = np.asarray(np.sum(a, axis=axis))
            assert ora.reduce_sum(a, axis).tobytes() == want.tobytes(), axis
            assert _planned_sum(a, axis).tobytes() == want.reshape(-1).tobytes(), axis


@pytest.mark.parametrize("dtypes", [(np.float64, np.float64), (np.float32, np.float64), (np.float32, np.float32)])
@pytest.mark.parametrize("conditioning", [None, "single", "double"])
def test_oracle_nanmean_sums_match_numpy(dtypes, conditioning):
    rng = np.random.default_rng(7)
    pred = _data(rng, (6, 1, 40, 33), dtypes[0])
    obs = _data(rng, (6, 1, 40, 33), dtypes[1])
    pred[rng.random(pred.shape) < 0.1] = np.nan
    obs[rng.random(obs.shape) < 0.05] = np.inf
    for axis in [(0,), (2, 3), (0, 2), (0, 1, 2, 3), (1,)]:
        tot, cnt, n = ora.cont_sums(pred, obs, axis, conditioning, 0.5)
        p, o = pred.copy(), obs.copy()
        if conditioning:
            keep = (o > 0.5) | (p > 0.5) if conditioning == "single" else (o > 0.5) & (p > 0.5)
            p[~keep], o[~keep] = np.nan, np.nan
        with np.errstate(all="ignore"), np.testing.suppress_warnings() as sup:
            sup.filter(RuntimeWarning)
            res, s = p - o, p + o
            means = [np.nanmean(x, axis=axis) for x in (o, p, res, res ** 2, s ** 2, np.abs(res))]
            mo, mp = means[0], means[1]
            for ax in sorted(axis):
                mo, mp = np.expand_dims(mo, ax), np.expand_dims(mp, ax)
            means += [np.nanmean(x, axis=axis) for x in ((o - mo) * (p - mp), np.abs(o - mo) ** 2, np.abs(p - mp) ** 2)]
            got = [(t.astype(np.float64) / c).astype(m.dtype) for t, c, m in zip(tot, cnt, means)]
        for k, (g, m) in enumerate(zip(got, means)):
            assert g.tobytes() == np.asarray(m).tobytes(), (axis, k)
        assert np.array_equal(n, np.sum(np.isfinite(res), axis=axis))
