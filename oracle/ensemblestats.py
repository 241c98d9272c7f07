"""Oracle of the ensemble statistics (pysteps/postprocessing/ensemblestats.py:20-179).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Restates mean, excprob and banddepth with
explicit loops over the members and integer counts, in the arithmetic the device uses:
  * mean: the sequential sum over members in X's dtype, starting from 0, divided by k; nanmean adds
    0 for every NaN (and, with X_thr, every value below it) and divides float64(sum) by the count
  * excprob: exact counts of finite members >= each threshold, over k or over the finite members
  * banddepth: each member's rank 1 + #{j : (X_j, b_j) < (X_i, b_i)} with the lower member index
    winning a full tie, the int64 sums of (k - rank) (rank - 1), and the reference's float64 tail
NumPy computes the same values wherever the member axis is outermost in memory (its reduction over
that axis is sequential).  Thresholds are compared in ``np.result_type(X, threshold)`` (NEP 50).
These functions return values only: the argument checks and warnings are the host's.
"""
import numpy as np
from scipy.special import comb


def _cmp(X, thr):
    """thr as the float NumPy compares X with (float64, after rounding to the comparison dtype)"""
    ct = np.result_type(X, thr)
    return float(np.asarray(thr).astype(ct))


def mean(X, ignore_nan=False, X_thr=None):
    """X (k, m, n) or (m, n) float32/float64 -> (m, n) of X's dtype"""
    with np.errstate(all="ignore"):
        return _mean(X, ignore_nan, X_thr)


def _mean(X, ignore_nan, X_thr):
    X = np.asarray(X)
    if X.ndim == 2:
        X = X[None]
    k = X.shape[0]
    dt = X.dtype.type
    acc = np.zeros(X.shape[1:], dtype=dt)
    if not (ignore_nan or X_thr is not None):
        for i in range(k):
            acc = acc + X[i]
        return acc / dt(k)
    t = None if X_thr is None else _cmp(X, X_thr)
    cnt = np.zeros(X.shape[1:], dtype=np.int64)
    for i in range(k):
        drop = np.isnan(X[i])
        if t is not None:
            drop |= X[i].astype(np.float64) < t
        acc = acc + np.where(drop, dt(0), X[i])
        cnt += ~drop
    return (acc.astype(np.float64) / cnt).astype(dt)


def excprob(X, X_thr, ignore_nan=False):
    """X (k, ...) -> (len(X_thr), ...) float64, or (...) for a scalar threshold"""
    X = np.asarray(X)
    k = X.shape[0]
    scalar = np.isscalar(X_thr)
    thrs = [X_thr] if scalar else list(X_thr)
    finite = np.zeros(X.shape[1:], dtype=np.int64)
    for i in range(k):
        finite += np.isfinite(X[i])
    out = []
    for x in thrs:
        t = _cmp(X, x)
        cnt = np.zeros(X.shape[1:], dtype=np.int64)
        for i in range(k):
            cnt += np.isfinite(X[i]) & (X[i].astype(np.float64) >= t)
        with np.errstate(all="ignore"):
            if ignore_nan:
                P = cnt.astype(np.float64) / finite
            else:
                P = np.where(finite < k, np.nan, cnt.astype(np.float64) / k)
        out.append(P)
    return out[0] if scalar else np.stack(out)


def band_mask(X, thr):
    """(mask, col): the pixels (flattened in C order) whose members are all finite and some member
    >= thr, and each masked pixel's column (-1 elsewhere)"""
    X = np.asarray(X)
    k = X.shape[0]
    Xf = X.reshape(k, int(np.prod(X.shape[1:])))
    t = _cmp(X, thr)
    mask = np.ones(Xf.shape[1], dtype=bool)
    above = np.zeros(Xf.shape[1], dtype=bool)
    for i in range(k):
        mask &= np.isfinite(Xf[i])
        above |= Xf[i].astype(np.float64) >= t
    mask &= above
    col = np.full(Xf.shape[1], -1, dtype=np.int64)
    col[mask] = np.arange(int(mask.sum()))
    return mask, col


def band_match(X, mask, b):
    """(k,) int64: sum over the masked pixels of (k - rank) (rank - 1), b (k, p) the tie-breaks"""
    X = np.asarray(X)
    k = X.shape[0]
    V = X.reshape(k, int(np.prod(X.shape[1:])))[:, mask]
    match = np.zeros(k, dtype=np.int64)
    for i in range(k):
        r = np.ones(V.shape[1], dtype=np.int64)
        for j in range(k):
            if j == i:
                continue
            less = (V[j] < V[i]) | ((V[j] == V[i]) & ((b[j] < b[i]) | ((b[j] == b[i]) & (j < i))))
            r += less
        match[i] = int(((k - r) * (r - 1)).sum())
    return match


def banddepth(X, b, thr=None, norm=False):
    """The reference's depths with the tie-breaks b (k, p) given, p the number of masked pixels."""
    X = np.asarray(X)
    if thr is None:
        thr = np.nanmin(X)
    mask, _ = band_mask(X, thr)
    n = X.shape[0]
    p = np.sum(mask)
    assert b.shape == (n, p), (b.shape, n, p)
    match = band_match(X, mask, b)
    nchoose2 = comb(n, 2)
    proportion = match / p
    depth = (proportion + n - 1) / nchoose2
    if norm:
        depth = (depth - depth.min()) / (depth.max() - depth.min())
    return depth
