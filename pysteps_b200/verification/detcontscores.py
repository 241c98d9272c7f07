"""B200 continuous verification scores -- drop-in for the online scores of
``pysteps.verification.detcontscores``: ``det_cont_fct`` and its ``det_cont_fct_init`` / ``_accum`` /
``_merge`` / ``_compute`` steps.

``det_cont_fct_accum`` computes on the device (csrc/detscores.cu) what the reference's nine
``np.nanmean`` calls compute: the means of obs, pred, the residual, its square and absolute value, the
squared sum, and the centred products, each over its own non-NaN count, with every sum in NumPy's
order (``_reduction.plan``), and the count of finite residuals.  The host divides as NumPy divides,
raises NumPy's warnings in the reference's order ("Mean of empty slice", and the overflow and invalid
warnings of the element-wise operations and reductions), and applies the reference's parallel mean,
variance and covariance updates to the dict, so that dicts pass between the two packages both ways.
Two limits: a reduction that sums an infinity and also overflows to the same infinity elsewhere does
not report the overflow, and an axis tuple NumPy rejects (a repeated axis) raises NumPy's exception
without the warnings of the reference's element-wise operations before it.

The offline scores "scatter" and "corr_s", and ``scores=""`` which includes them, are not built on
the device and raise NotImplementedError; ``det_cont_fct_compute`` takes "" (its scores are all
online).  Inputs are NumPy arrays or CUDA tensors of float32 or float64 with at most 4 dimensions and
fewer than 2^31 elements.
"""
import warnings

import numpy as np
import torch

from .. import _device, _lib
from . import _inputs, _reduction
from .detcatscores import axis_tuple, check_array, score_names

_OFFLINE = ("scatter", "corr_s")
with np.errstate(invalid="ignore"):
    _HOST_NAN = np.float64(np.inf) - np.float64(np.inf)  # the NaN this host's float arithmetic makes
_KEYS = ("cov", "vobs", "vpred", "mobs", "mpred", "me", "mse", "mss", "mae", "n")


def _unique(names):
    seen, out = set(), []
    for x in names:
        if x not in seen:
            seen.add(x)
            out.append(x)
    return out


def det_cont_fct(pred, obs, scores="", axis=None, conditioning=None, thr=0.0):
    """The continuous scores `scores` (a list of online score names) of pred against obs."""
    scores = score_names(scores)
    online = _unique([s for s in scores if str(s).lower() not in _OFFLINE or s == ""])
    offline = _unique([s for s in scores if str(s).lower() in _OFFLINE or s == ""])
    if offline:
        raise NotImplementedError("pysteps_b200 det_cont_fct: the offline scores 'scatter' and 'corr_s' (and "
                                  "scores='', which includes them) are not built on the device; pass the online "
                                  "scores by name or use pysteps.verification.det_cont_fct")
    if not online:
        return {}
    err = det_cont_fct_init(axis=axis, conditioning=conditioning, thr=thr)
    det_cont_fct_accum(err, pred, obs)
    return det_cont_fct_compute(err, online)


def det_cont_fct_init(axis=None, conditioning=None, thr=0.0):
    """An empty verification error object."""
    err = {"axis": axis_tuple(axis), "conditioning": conditioning, "thr": thr}
    err.update(dict.fromkeys(_KEYS))
    return err


def host_nan(tot):
    """tot with every NaN written as this host's: a sum the device makes NaN has met +inf and -inf,
    and the GPU encodes inf - inf differently from the CPU NumPy runs on (x86: the negative quiet NaN,
    which then propagates through every later addition)"""
    tot[np.isnan(tot)] = _HOST_NAN
    return tot


def _warn(msg):
    warnings.warn(msg, RuntimeWarning, stacklevel=3)


def det_cont_fct_accum(err, pred, obs):
    """Add the moments of pred and obs to the verification error object."""
    who = "det_cont_fct_accum"
    check_array(pred, who, "pred")
    check_array(obs, who, "obs")
    shape, oshape = tuple(int(s) for s in pred.shape), tuple(int(s) for s in obs.shape)
    if shape != oshape:
        raise ValueError("the shape of pred does not match the shape of obs %s!=%s" % (shape, oshape))
    nshape, axis = _reduction.kept_shape(shape, err["axis"])
    pdt, odt = _inputs.np_dtype(pred), _inputs.np_dtype(obs)
    if err["cov"] is None:
        for key in _KEYS:
            err[key] = np.zeros(nshape)
    elif err["cov"].shape != nshape:
        raise ValueError("the shape of the input arrays does not match the shape of the verification object %s!=%s"
                         % (nshape, err["cov"].shape))
    cond, thr_p, thr_o = 0, 0.0, 0.0
    if err["conditioning"] is not None:
        if err["conditioning"] == "single":
            cond = 1
        elif err["conditioning"] == "double":
            cond = 2
        else:
            raise ValueError("unkown conditioning %s" % err["conditioning"])
        thr_p, thr_o = _inputs.threshold(pdt, err["thr"], who), _inputs.threshold(odt, err["thr"], who)
    eshape, eaxis = _reduction.effective(shape, axis)
    M = _inputs.pixels(nshape)
    tot, cnt = np.zeros((9, M)), np.zeros((10, M), np.int64)
    infs, flags = np.zeros(M, np.int32), 0
    if M and _inputs.pixels(eshape):
        (ks, kst), (os_, ost), L = _reduction.plan(eshape, eaxis)
        p = _inputs.to_device(pred, (-1,))
        o = _inputs.to_device(obs, (-1,))
        d_tot = torch.empty(9 * M, dtype=torch.float64, device="cuda")
        d_cnt = torch.empty(10 * M, dtype=torch.int64, device="cuda")
        d_infs = torch.empty(M, dtype=torch.int32, device="cuda")
        d_flags = torch.empty(1, dtype=torch.int32, device="cuda")
        _lib.call("b200_verif_cont_moments", p.data_ptr(), _device.dtype_code(p.dtype), o.data_ptr(),
                  _device.dtype_code(o.dtype), cond, thr_p, thr_o, *_reduction.c_axes(ks, kst),
                  *_reduction.c_axes(os_, ost), L, d_tot.data_ptr(), d_cnt.data_ptr(), d_infs.data_ptr(),
                  d_flags.data_ptr(), _device.stream_ptr())
        tot, cnt = host_nan(_device.to_host(d_tot).reshape(9, M)), _device.to_host(d_cnt).reshape(10, M)
        infs, flags = _device.to_host(d_infs), int(_device.to_host(d_flags)[0])
    _finish(err, nshape, eaxis, [odt, pdt] + [np.result_type(pdt, odt)] * 5 + [odt, pdt], tot, cnt, infs, flags)


def _finish(err, nshape, axis, dtypes, tot, cnt, infs, flags):
    """the reference's nine np.nanmean results and warnings from the device's sums, then its updates"""
    scalar = nshape == ()

    def elementwise(op, over, inv=0):
        if flags & over:
            _warn(f"overflow encountered in {op}")
        if flags & inv:
            _warn(f"invalid value encountered in {op}")

    def nanmean(k):
        t, c, dt = tot[k], cnt[1 + k], dtypes[k]
        pos, neg = (infs >> (2 * k)) & 1 == 1, (infs >> (2 * k + 1)) & 1 == 1
        nan = np.isnan(t)
        if (((~np.isfinite(t)) & ~pos & ~neg) | (nan & ~(pos & neg))).any():
            _warn("overflow encountered in reduce")
        if nan.any():
            _warn("invalid value encountered in reduce")
        with np.errstate(invalid="ignore", divide="ignore"):
            if scalar:
                mean = dt.type(dt.type(t[0]) / np.intp(c[0]))
            else:
                mean = t.astype(dt).reshape(nshape)
                np.true_divide(mean, c.astype(np.intp).reshape(nshape), out=mean, casting="unsafe")
        if (c == 0).any():
            _warn("Mean of empty slice")
        return mean

    elementwise("subtract", _lib.MOM_SUB_RES_OVER, _lib.MOM_SUB_RES_INV)
    elementwise("add", _lib.MOM_ADD_SUM_OVER, _lib.MOM_ADD_SUM_INV)
    n = np.intp(cnt[0, 0]) if scalar else cnt[0].astype(np.intp).reshape(nshape)
    mobs, mpred, me = nanmean(0), nanmean(1), nanmean(2)
    elementwise("square", _lib.MOM_SQ_RES_OVER)
    mse = nanmean(3)
    elementwise("square", _lib.MOM_SQ_SUM_OVER)
    mss = nanmean(4)
    mae = nanmean(5)
    for ax in sorted(axis):
        mobs, mpred = np.expand_dims(mobs, ax), np.expand_dims(mpred, ax)
    elementwise("subtract", _lib.MOM_SUB_OBS_OVER, _lib.MOM_SUB_OBS_INV)
    elementwise("subtract", _lib.MOM_SUB_PRED_OVER, _lib.MOM_SUB_PRED_INV)
    elementwise("multiply", _lib.MOM_MUL_OVER, _lib.MOM_MUL_INV)
    cov = nanmean(6)
    elementwise("subtract", _lib.MOM_SUB_OBS_OVER, _lib.MOM_SUB_OBS_INV)
    elementwise("square", _lib.MOM_SQ_VOBS_OVER)
    vobs = nanmean(7)
    elementwise("subtract", _lib.MOM_SUB_PRED_OVER, _lib.MOM_SUB_PRED_INV)
    elementwise("square", _lib.MOM_SQ_VPRED_OVER)
    vpred = nanmean(8)
    mobs, mpred = mobs.squeeze(), mpred.squeeze()
    _update(err, dict(mobs=mobs, mpred=mpred, vobs=vobs, vpred=vpred, cov=cov, me=me, mse=mse, mss=mss, mae=mae, n=n))


def _update(err, new):
    """merge the moments `new` into err in place: Chan et al.'s parallel variance and covariance, then
    the count-weighted means, where new["n"] > 0"""
    n_a, n_b = err["n"], new["n"]
    _merge_var(err["mobs"], n_a, err["vobs"], new["mobs"], n_b, new["vobs"])
    _merge_var(err["mpred"], n_a, err["vpred"], new["mpred"], n_b, new["vpred"])
    _merge_cov(err["cov"], err["mobs"], err["mpred"], n_a, new["cov"], new["mobs"], new["mpred"], n_b)
    for key in ("mobs", "mpred", "me", "mse", "mss", "mae"):
        _merge_mean(err[key], n_a, new[key], n_b)
    err["n"] += n_b


def _merge_mean(mean_a, n_a, mean_b, n_b):
    sel = n_b > 0
    mean_a[sel] = (n_a[sel] * mean_a[sel] + n_b[sel] * mean_b[sel]) / (n_a[sel] + n_b[sel])


def _merge_var(mean_a, n_a, var_a, mean_b, n_b, var_b):
    sel = n_b > 0
    delta = mean_b - mean_a
    sq_a, sq_b = var_a * n_a, var_b * n_b
    var_a[sel] = sq_a[sel] + sq_b[sel] + delta[sel] ** 2 * n_a[sel] * n_b[sel] / (n_a[sel] + n_b[sel])
    var_a[sel] = var_a[sel] / (n_a[sel] + n_b[sel])


def _merge_cov(cov_a, mx_a, my_a, n_a, cov_b, mx_b, my_b, n_b):
    sel = n_b > 0
    dx, dy = mx_b - mx_a, my_b - my_a
    c_a, c_b = cov_a * n_a, cov_b * n_b
    cov_a[sel] = c_a[sel] + c_b[sel] + dx[sel] * dy[sel] * n_a[sel] * n_b[sel] / (n_a[sel] + n_b[sel])
    cov_a[sel] = cov_a[sel] / (n_a[sel] + n_b[sel])


def det_cont_fct_merge(err_1, err_2):
    """err_1 with the moments of err_2 merged in (a shallow copy: err_1's arrays are updated in place,
    as in the reference)."""
    for key, what in (("axis", "axis are"), ("conditioning", "conditioning is"), ("thr", "threshold is")):
        if err_1[key] != err_2[key]:
            raise ValueError("cannot merge: the %s not same %s!=%s" % (what, err_1[key], err_2[key]))
    if err_1["cov"] is None or err_2["cov"] is None:
        raise ValueError("cannot merge: no data found")
    err = err_1.copy()
    _update(err, err_2)
    return err


def det_cont_fct_compute(err, scores=""):
    """The online scores of the error object: "" for all, or any of beta (beta1), beta2, corr_p
    (pearsonr), drmse, mae, me (bias), mse, nmse, rmse, rv (brier_score, nse), case-insensitive."""
    result = {}
    for score in score_names(scores):
        if score is None:
            continue
        name = score.lower()
        if name in ("bias", "me", ""):
            result["ME"] = err["me"]
        if name in ("mae", ""):
            result["MAE"] = err["mae"]
        if name in ("mse", ""):
            result["MSE"] = err["mse"]
        if name in ("nmse", ""):
            result["NMSE"] = err["mse"] / err["mss"]
        if name in ("rmse", ""):
            result["RMSE"] = np.sqrt(err["mse"])
        if name in ("corr_p", "pearsonr", ""):
            result["corr_p"] = err["cov"] / np.sqrt(err["vobs"]) / np.sqrt(err["vpred"])
        if name in ("beta", "beta1", ""):
            result["beta1"] = err["cov"] / err["vpred"]
        if name in ("beta2", ""):
            result["beta2"] = err["cov"] / err["vobs"]
        if name in ("drmse", ""):
            result["DRMSE"] = np.sqrt(err["mse"] - err["me"] ** 2)
        if name in ("rv", "brier_score", "nse", ""):
            result["RV"] = 1.0 - err["mse"] / err["vobs"]
    return result
