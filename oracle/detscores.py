"""CPU ORACLE of the deterministic and spatial verification accumulators of
pysteps/verification/detcatscores.py, spatialscores.py and ensscores.py, restated in plain NumPy without
the reference's code:

    contab(pred, obs, thr, axis)       -> (hits, false_alarms, misses, correct_negatives) as int64 arrays of
                                          the kept axes, axis a tuple of non-negative axes
    uniform_filter(I, s)               -> scipy.ndimage.uniform_filter(I, size=s, mode="constant") restated:
                                          the running sum along axis 0, then along axis 1
    fractions(X, thr, scale)           -> the smoothed indicator of fss_accum (float64)
    fss_sums(X_f, X_o, thr, scale)     -> (sum_obs_sq, sum_fct_obs, sum_fct_sq) that fss_accum adds
    spread_fss(X_f, thr, scale)        -> the FSS of every member pair (i < j), in the reference's order
    reduce_sum(a, axis)                -> np.sum(a, axis) of a C-contiguous float array, restated
    cont_sums(pred, obs, axis, conditioning, thr)
                                       -> (tot, cnt, n): the nine sums det_cont_fct_accum's np.nanmean
                                          calls take (NaN as 0) and their non-NaN counts, and the count
                                          of finite residuals, over the non-negative axes `axis`

np.sum(a, axis) of a C-contiguous float array, size-1 axes aside: every output element starts at 0
and adds, for each index of the reduced axes left of a kept axis (in C order), the pairwise sum of the
trailing run of reduced axes taken as one contiguous run.
"""
import numpy as np

from .verification import _threshold, pairwise


def contab(pred, obs, thr, axis):
    pred, obs = np.asarray(pred), np.asarray(obs)
    kept = [d for d in range(pred.ndim) if d not in axis]
    order = kept + sorted(axis)
    p = np.transpose(pred, order).reshape([pred.shape[d] for d in kept] + [-1])
    o = np.transpose(obs, order).reshape(p.shape)
    pb = p.astype(np.float64) > _threshold(pred.dtype, thr)
    ob = o.astype(np.float64) > _threshold(obs.dtype, thr)
    return tuple((c.sum(axis=-1, dtype=np.int64)) for c in (pb & ob, pb & ~ob, ~pb & ob, ~pb & ~ob))


def _running(X, s):
    """scipy's 1-D uniform filter along the last axis: s // 2 zeros in front, the first window summed
    left to right, then tmp += (entering - leaving) and out = tmp / s"""
    L = X.shape[-1]
    s1 = s // 2
    pad = np.concatenate([np.zeros(X.shape[:-1] + (s1,)), X, np.zeros(X.shape[:-1] + (s,))], axis=-1)
    out = np.empty(X.shape, dtype=np.float64)
    tmp = np.zeros(X.shape[:-1])
    for j in range(s):
        tmp = tmp + pad[..., j]
    out[..., 0] = tmp / float(s)
    for j in range(1, L):
        tmp = tmp + (pad[..., j + s - 1] - pad[..., j - 1])
        out[..., j] = tmp / float(s)
    return out


def uniform_filter(I, s):
    return _running(_running(np.asarray(I, dtype=np.float64).T, s).T, s)


def fractions(X, thr, scale):
    X = np.asarray(X)
    sub = np.asarray(thr - 1).astype(X.dtype)
    X = np.where(np.isfinite(X), X, sub)
    I = (X.astype(np.float64) >= _threshold(X.dtype, thr)).astype(np.float64)
    s = int(scale) if scale > 1 else 1
    if s <= 1 or I.size == 0:
        return I
    return uniform_filter(I, s)


def _psum(a):
    return pairwise(np.ascontiguousarray(a).reshape(-1))


def fss_sums(X_f, X_o, thr, scale):
    S_f, S_o = fractions(X_f, thr, scale), fractions(X_o, thr, scale)
    return _psum(S_o * S_o), _psum(S_f * S_o), _psum(S_f * S_f)


def _fss(oo, fo, ff):
    return 1.0 - (ff - 2.0 * fo + oo) / (ff + oo)


def spread_fss(X_f, thr, scale):
    S = [fractions(x, thr, scale) for x in X_f]
    out = []
    for i in range(len(S)):
        for j in range(i + 1, len(S)):
            with np.errstate(invalid="ignore", divide="ignore"):
                out.append(_fss(_psum(S[j] * S[j]), _psum(S[i] * S[j]), _psum(S[i] * S[i])))
    return out


def reduce_sum(a, axis):
    a = np.asarray(a)
    axis = tuple(axis)
    out_shape = tuple(a.shape[d] for d in range(a.ndim) if d not in axis)
    dims = [d for d in range(a.ndim) if a.shape[d] != 1]
    t = len(dims)
    while t > 0 and dims[t - 1] in axis:
        t -= 1
    kept = [d for d in dims[:t] if d not in axis]
    outer = [d for d in dims[:t] if d in axis]
    inner = dims[t:]
    b = np.transpose(a.reshape([a.shape[d] for d in dims]), [dims.index(d) for d in kept + outer + inner])
    K = int(np.prod([a.shape[d] for d in kept], dtype=np.int64))
    O = int(np.prod([a.shape[d] for d in outer], dtype=np.int64))
    b = np.ascontiguousarray(b).reshape(K, O, -1)
    part = pairwise(b) if b.shape[-1] else np.zeros((K, O), a.dtype)
    out = np.zeros(K, a.dtype)
    for o in range(O):
        out = out + part[:, o]
    return out.reshape(out_shape)


def cont_sums(pred, obs, axis, conditioning, thr):
    pred, obs = np.asarray(pred), np.asarray(obs)
    if conditioning is not None:
        sp = pred.astype(np.float64) > _threshold(pred.dtype, thr)
        so = obs.astype(np.float64) > _threshold(obs.dtype, thr)
        keep = (sp | so) if conditioning == "single" else (sp & so)
        pred, obs = np.where(keep, pred, np.nan).astype(pred.dtype), np.where(keep, obs, np.nan).astype(obs.dtype)
    R = np.result_type(pred.dtype, obs.dtype)
    with np.errstate(all="ignore"):
        res = pred.astype(R) - obs.astype(R)
        tot_ = pred.astype(R) + obs.astype(R)
        first = [obs, pred, res, res * res, tot_ * tot_, np.abs(res)]
        tot = [reduce_sum(np.where(np.isnan(x), x.dtype.type(0), x), axis) for x in first]
        cnt = [reduce_sum((~np.isnan(x)).astype(np.int64), axis) for x in first]
        n = reduce_sum(np.isfinite(res).astype(np.int64), axis)
        mo = (tot[0].astype(np.float64) / cnt[0]).astype(obs.dtype)
        mp = (tot[1].astype(np.float64) / cnt[1]).astype(pred.dtype)
        for ax in sorted(axis):
            mo, mp = np.expand_dims(mo, ax), np.expand_dims(mp, ax)
        dq, dp = obs - mo, pred - mp
        second = [dq.astype(R) * dp.astype(R), np.abs(dq) * np.abs(dq), np.abs(dp) * np.abs(dp)]
        tot += [reduce_sum(np.where(np.isnan(x), x.dtype.type(0), x), axis) for x in second]
        cnt += [reduce_sum((~np.isnan(x)).astype(np.int64), axis) for x in second]
    return tot, cnt, n
