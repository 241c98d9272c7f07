"""The deterministic and spatial verification scores on the device (pysteps_b200.verification's
detcatscores, detcontscores, spatialscores and the ensemble skill and spread) against the stored
reference outcomes, the oracle (oracle/detscores.py) and NumPy's own np.nanmean: every golden call bit
for bit with its warnings, 2048^2 fields in float32 and float64 as NumPy arrays and CUDA tensors,
12-step stacks, 24-member FSS skill and spread against the per-member and per-pair ``fss`` calls, and
the calls refused before any launch."""
import os
from unittest import mock

import numpy as np
import pytest
import torch

from detscores_cases import field, golden_calls, numpy_moments, our_modules, run_call
from oracle import detscores as ora
from verification_cases import Goldens, matches_golden

pytestmark = pytest.mark.gpu
GOLDEN = Goldens(os.path.join(os.path.dirname(__file__), "golden", "detscores_golden.npz"))
CALLS = golden_calls()
KEYS = ("hits", "false_alarms", "misses", "correct_negatives")


@pytest.mark.parametrize("i", range(len(CALLS)), ids=[c[0] for c in CALLS])
def test_golden_calls(i):
    key, mod, fn, args, kwargs = CALLS[i]
    out, warned = run_call(our_modules()[mod], fn, args, kwargs)
    problems = matches_golden(GOLDEN, key, out, warned, None)
    assert not problems, (key, problems)


def _bits(x):
    return np.asarray(x, dtype=np.float64).tobytes()


@pytest.fixture(scope="module")
def big():
    rng = np.random.default_rng(31)
    X = field(rng, (2048, 2048), nans=0.01, infs=0.001)
    Y = np.where(rng.random((2048, 2048)) < 0.3, X, field(rng, (2048, 2048), nans=0.01))
    return X, Y


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("tensor", [False, True])
def test_contab_2048(big, dtype, tensor):
    from pysteps_b200 import verification as v
    X, Y = (a.astype(dtype) for a in big)
    x, y = (torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()) if tensor else (X, Y)
    for axis in (None, -1, 0, 1):
        eff = (0, 1) if axis is None else ((0,) if axis == -1 else (axis,))
        want = ora.contab(X[None] if axis == -1 else X, Y[None] if axis == -1 else Y, 1.0, eff)
        for _ in range(2):  # repeated calls are identical
            c = v.det_cat_fct_init(1.0, axis)
            v.det_cat_fct_accum(c, x, y)
            for key, w in zip(KEYS, want):
                assert np.array_equal(c[key], w), (axis, key)


@pytest.mark.parametrize("axis", [(1, 2), 0])
def test_contab_12_steps(axis):
    from pysteps_b200 import verification as v
    rng = np.random.default_rng(32)
    X = field(rng, (12, 2048, 2048), np.float32, nans=0.01)
    Y = field(rng, (12, 2048, 2048), np.float32, nans=0.01)
    c = v.det_cat_fct_init(0.5, axis)
    v.det_cat_fct_accum(c, torch.from_numpy(X).cuda(), Y)
    want = ora.contab(X, Y, 0.5, axis if isinstance(axis, tuple) else (axis,))
    for key, w in zip(KEYS, want):
        assert np.array_equal(c[key], w), key


def _device_moments(pred, obs, axis, cond, thr):
    """the nine means and the finite count of b200_verif_cont_moments, divided as NumPy divides"""
    from pysteps_b200 import _device, _lib
    from pysteps_b200.verification import _inputs, _reduction, detcontscores
    shape = tuple(pred.shape)
    kept = tuple(shape[d] for d in range(len(shape)) if d not in axis)
    (ks, kst), (os_, ost), L = _reduction.plan(shape, axis)
    M = int(np.prod(kept, dtype=np.int64))
    pdt, odt = _inputs.np_dtype(pred), _inputs.np_dtype(obs)
    code = {None: 0, "single": 1, "double": 2}[cond]
    p, o = _inputs.to_device(pred, (-1,)), _inputs.to_device(obs, (-1,))
    tot = torch.empty(9 * M, dtype=torch.float64, device="cuda")
    cnt = torch.empty(10 * M, dtype=torch.int64, device="cuda")
    infs = torch.empty(M, dtype=torch.int32, device="cuda")
    flags = torch.empty(1, dtype=torch.int32, device="cuda")
    _lib.call("b200_verif_cont_moments", p.data_ptr(), _device.dtype_code(p.dtype), o.data_ptr(),
              _device.dtype_code(o.dtype), code, _inputs.threshold(pdt, thr, "t"), _inputs.threshold(odt, thr, "t"),
              *_reduction.c_axes(ks, kst), *_reduction.c_axes(os_, ost), L, tot.data_ptr(), cnt.data_ptr(),
              infs.data_ptr(), flags.data_ptr(), _device.stream_ptr())
    t, c = detcontscores.host_nan(_device.to_host(tot).reshape(9, M)), _device.to_host(cnt).reshape(10, M)
    R = np.result_type(pdt, odt)
    dts = [odt, pdt, R, R, R, R, R, odt, pdt]
    with np.errstate(all="ignore"):
        means = [(t[k] / c[1 + k]).astype(dts[k]).reshape(kept) for k in range(9)]
    return means, c[0].reshape(kept)


def _same_moments(got, want):
    for k, (g, w) in enumerate(zip(got[0], want[0])):
        assert g.tobytes() == np.asarray(w).tobytes(), k
    assert np.array_equal(got[1], want[1])


@pytest.mark.parametrize("dtypes", [(np.float32, np.float32), (np.float64, np.float32), (np.float64, np.float64)])
@pytest.mark.parametrize("tensor", [False, True])
def test_moments_2048(big, dtypes, tensor):
    X, Y = big[0].astype(dtypes[0]), big[1].astype(dtypes[1])
    x, y = (torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()) if tensor else (X, Y)
    for axis, cond in (((0, 1), None), ((0,), None), ((1,), "double"), ((0, 1), "single")):
        want = numpy_moments(X, Y, axis, cond, 0.5)
        for _ in range(2):
            _same_moments(_device_moments(x, y, axis, cond, 0.5), want)
    # no integration: the leading unit axis the reference adds
    _same_moments(_device_moments(x[None], y[None], (0,), None, 0.5), numpy_moments(X[None], Y[None], (0,), None, 0.5))


@pytest.mark.parametrize("axis", [(1, 2), (0,)])
def test_moments_12_steps(axis):
    rng = np.random.default_rng(36)
    X = field(rng, (12, 2048, 2048), np.float32, nans=0.01)
    Y = field(rng, (12, 2048, 2048), np.float32, nans=0.01, infs=0.0001)
    _same_moments(_device_moments(torch.from_numpy(X).cuda(), Y, axis, None, 0.5), numpy_moments(X, Y, axis, None, 0.5))


def test_det_cont_fct_tensor_equals_numpy():
    from pysteps_b200 import verification as v
    rng = np.random.default_rng(37)
    X, Y = field(rng, (3, 512, 384), nans=0.02), field(rng, (3, 512, 384), np.float32, nans=0.02)
    scores = ["ME", "MAE", "MSE", "NMSE", "RMSE", "corr_p", "beta1", "beta2", "DRMSE", "RV"]
    a = v.det_cont_fct(X, Y, scores, axis=(1, 2), conditioning="single", thr=0.3)
    b = v.det_cont_fct(torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda(), scores, axis=(1, 2),
                       conditioning="single", thr=0.3)
    assert list(a) == scores
    assert all(a[k].tobytes() == b[k].tobytes() for k in a)


def _fss_sums(X_f, X_o, thr, scale):
    """the oracle's fractions with NumPy's own pairwise sum (the oracle's restatement of it is pinned
    to np.sum on the CPU; in Python it is too slow for 2048^2 planes)"""
    S_f, S_o = ora.fractions(X_f, thr, scale), ora.fractions(X_o, thr, scale)
    return np.sum(S_o * S_o), np.sum(S_f * S_o), np.sum(S_f * S_f)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("tensor", [False, True])
def test_fss_2048(big, dtype, tensor):
    from pysteps_b200 import verification as v
    X, Y = (a.astype(dtype) for a in big)
    x, y = (torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()) if tensor else (X, Y)
    for thr, scale in ((1.0, 16), (0.1, 1), (2.0, 3)):
        want = _fss_sums(X, Y, thr, scale)
        for _ in range(2):
            d = v.fss_init(thr, scale)
            v.fss_accum(d, x, y)
            got = (d["sum_obs_sq"], d["sum_fct_obs"], d["sum_fct_sq"])
            assert all(_bits(g) == _bits(w) for g, w in zip(got, want)), (thr, scale, got, want)


def test_fss_mixed_dtypes():
    from pysteps_b200 import verification as v
    rng = np.random.default_rng(33)
    X, Y = field(rng, (300, 257), np.float32, nans=0.02), field(rng, (300, 257), nans=0.02)
    d = v.fss_init(np.float32(0.7), 9)
    v.fss_accum(d, X, torch.from_numpy(Y).cuda())
    want = ora.fss_sums(X, Y, np.float32(0.7), 9)
    assert _bits([d["sum_obs_sq"], d["sum_fct_obs"], d["sum_fct_sq"]]) == _bits(want)


def test_spread_and_skill_against_the_oracle():
    from pysteps_b200 import verification as v
    rng = np.random.default_rng(34)
    E = field(rng, (19, 64, 48), nans=0.02)  # two member groups
    o = field(rng, (64, 48), np.float32)
    assert _bits(v.ensemble_spread(E, "fss", thr=1.0, scale=5)) == _bits(np.mean(ora.spread_fss(E, 1.0, 5)))
    want = []
    for x in E:
        oo, fo, ff = ora.fss_sums(x, o, 1.0, 5)
        want.append(1.0 - (ff - 2.0 * fo + oo) / (ff + oo))
    assert _bits(v.ensemble_skill(E, o, "fss", thr=1.0, scale=5)) == _bits(np.mean(want))


def test_24_members_batched_equals_per_pair_fss():
    from pysteps_b200 import verification as v
    rng = np.random.default_rng(35)
    E = torch.from_numpy(field(rng, (24, 2048, 2048), np.float32, nans=0.01)).cuda()
    o = torch.from_numpy(field(rng, (2048, 2048), np.float32, nans=0.01)).cuda()
    pairs = [v.fss(E[i], E[j], 1.0, 16) for i in range(24) for j in range(i + 1, 24)]
    assert _bits(v.ensemble_spread(E, "fss", thr=1.0, scale=16)) == _bits(np.mean(pairs))
    members = [v.fss(E[i], o, 1.0, 16) for i in range(24)]
    assert _bits(v.ensemble_skill(E, o, "fss", thr=1.0, scale=16)) == _bits(np.mean(members))


def test_refused_before_any_launch():
    from pysteps_b200 import _lib
    from pysteps_b200 import verification as v
    X = np.zeros((4, 5))
    refused = [
        (v.det_cat_fct, (X.astype(np.int64), X, 0.5)),
        (v.det_cat_fct, (np.ma.masked_array(X), X, 0.5)),
        (v.det_cat_fct, (torch.zeros(4, 5, dtype=torch.float64), X, 0.5)),
        (v.det_cat_fct, (np.zeros((1, 1, 1, 1, 2)), np.zeros((1, 1, 1, 1, 2)), 0.5)),
        (v.det_cat_fct, (X, X, "0.5")),
        (v.fss, (X.astype(np.int32), X, 0.5, 2)),
        (v.fss, (X, X, 0.5, 1 << 40)),
        (v.binary_mse, (X, X, 0.5)),
        (v.sal, (X, X)),
        (v.intensity_scale, (X, X, "BMSE", 0.5)),
        (v.ensemble_spread, (np.zeros((513, 2, 2)), "fss"), {"thr": 0.5, "scale": 2}),
        (v.ensemble_skill, (np.zeros((3, 2, 2)), X[:2, :2], "corr_s"), {}),
        (v.det_cont_fct, (X, X), {}),
        (v.det_cont_fct, (X, X, ["rmse", "scatter"]), {}),
        (v.det_cont_fct, (X.astype(np.float16), X, ["rmse"]), {}),
        (v.ensemble_spread, (np.zeros((3, 2, 2)), "sal"), {}),
        (v.det_cat_fct, (np.broadcast_to(np.float32(0), (1 << 31,)), np.broadcast_to(np.float32(0), (1 << 31,)), 0.5)),
    ]
    with mock.patch.object(_lib, "call", side_effect=AssertionError("launched")):
        for fn, args, *kw in refused:
            with pytest.raises(NotImplementedError):
                fn(*args, **(kw[0] if kw else {}))
