"""CPU ORACLE of the verification accumulators of pysteps/verification/probscores.py and ensscores.py,
restated in plain NumPy without the reference's code: an explicit restatement of NumPy's pairwise
summation, vectorised over rows, and exact integer counts.  Each function returns what its
``*_accum`` adds to the accumulator dict:

    crps(X_f, X_o)                    -> (sum of the per-pixel CRPS as np.float64, pixel count)
    crps_pixels(X_f, X_o)             -> the per-pixel CRPS of the finite pixels in pixel order
    crps_loop(X_f, X_o)               -> the same, one pixel and one column at a time in Python
    rankhist(X_f, X_o, X_min, u=None) -> (bin counts without the ties, (b1, b2) of the tied pixels)
                                         and, given the draws u, the full counts
    reldiag(P_f, X_o, X_min, edges)   -> (count, count of X_o >= X_min, pairwise sum of P_f) per bin
    roc(P_f, X_o, X_min, thrs)        -> (hits, misses, false_alarms, corr_neg) per threshold
"""
import numpy as np


def pairwise(a):
    """np.sum(a, axis=-1) of a C-contiguous array, restated: 0 + pw(a) in a's dtype"""
    a = np.asarray(a)
    zero = np.zeros(a.shape[:-1], dtype=a.dtype)
    return zero + _pw(a, 0, a.shape[-1], zero)


def _pw(a, lo, n, zero):
    if n < 8:
        r = zero.copy()
        for i in range(n):
            r = r + a[..., lo + i]
        return r
    if n <= 128:
        r = [a[..., lo + j].copy() for j in range(8)]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = r[j] + a[..., lo + i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for t in range(i, n):
            res = res + a[..., lo + t]
        return res
    h = n // 2
    h -= h % 8
    return _pw(a, lo, h, zero) + _pw(a, lo + h, n - h, zero)


def _layout(X_f, X_o):
    k = X_f.shape[0]
    return np.asarray(X_f).reshape(k, -1).T, np.asarray(X_o).reshape(-1)


def crps(X_f, X_o):
    per_pixel = crps_pixels(X_f, X_o)
    return pairwise(per_pixel), int(len(per_pixel))


def crps_pixels(X_f, X_o):
    F, O = _layout(X_f, X_o)
    k = F.shape[1]
    keep = np.isfinite(F).all(axis=1) & np.isfinite(O)
    F = np.sort(F[keep], axis=1)
    O = O[keep]
    P = np.result_type(F.dtype, O.dtype)
    Fw, Ow = F.astype(P), O.astype(P)
    o = O.astype(np.float64)
    x = F.astype(np.float64)
    alpha = np.zeros((len(O), k + 1))
    beta = np.zeros((len(O), k + 1))
    for i in range(1, k):
        d = (F[:, i] - F[:, i - 1]).astype(np.float64)
        up = o > x[:, i]
        mid = (x[:, i] > o) & (o > x[:, i - 1])
        down = o < x[:, i - 1]
        alpha[:, i] = np.where(up, d, np.where(mid, (Ow - Fw[:, i - 1]).astype(np.float64), 0.0))
        beta[:, i] = np.where(mid, (Fw[:, i] - Ow).astype(np.float64), np.where(down, d, 0.0))
    first = o < x[:, 0]
    beta[:, 0] = np.where(first, (Fw[:, 0] - Ow).astype(np.float64), 0.0)
    last = x[:, k - 1] < o
    alpha[:, k] = np.where(last, (Ow - Fw[:, k - 1]).astype(np.float64), alpha[:, k])
    p = np.arange(k + 1, dtype=np.float64) / k
    terms = alpha * (p * p) + beta * ((1.0 - p) * (1.0 - p))
    return pairwise(np.ascontiguousarray(terms)) if len(O) else np.zeros(0)


def crps_loop(X_f, X_o):
    """crps_pixels from the definition, pixel by pixel: the area between the ensemble's step CDF and
    the observation's, as the k + 1 intervals of the sorted members weighted by p^2 below the
    observation and (1 - p)^2 above it; an interval that ends exactly at the observation counts
    nothing (the reference's strict comparisons)"""
    F, O = _layout(X_f, X_o)
    k = F.shape[1]
    P = np.result_type(F.dtype, O.dtype).type
    out = []
    for x, o in zip(F, O):
        if not (np.isfinite(x).all() and np.isfinite(o)):
            continue
        x = np.sort(x)
        terms = []
        for i in range(k + 1):
            p = np.float64(i) / k
            below = above = 0.0
            if i == 0:
                if o < x[0]:
                    above = float(P(x[0]) - P(o))
            elif i == k:
                if x[k - 1] < o:
                    below = float(P(o) - P(x[k - 1]))
            elif o > x[i]:
                below = float(x[i] - x[i - 1])
            elif x[i - 1] < o < x[i]:
                below, above = float(P(o) - P(x[i - 1])), float(P(x[i]) - P(o))
            elif o < x[i - 1]:
                above = float(x[i] - x[i - 1])
            terms.append(np.float64(below) * (p * p) + np.float64(above) * ((1.0 - p) * (1.0 - p)))
        out.append(pairwise(np.array(terms)))
    return np.array(out, dtype=np.float64)


def _threshold(dtype, X_min):
    ct = np.result_type(np.zeros(1, dtype=dtype), X_min)
    return np.asarray(X_min).astype(ct)


def rankhist(X_f, X_o, X_min=None, u=None):
    F, O = _layout(X_f, X_o)
    k = F.shape[1]
    keep = np.isfinite(F).all(axis=1) & np.isfinite(O)
    if X_min is not None:
        keep &= (O >= _threshold(O.dtype, X_min)) | (F >= _threshold(F.dtype, X_min)).any(axis=1)
    F, O = F[keep].copy(), O[keep].copy()
    if X_min is not None:
        F[F < _threshold(F.dtype, X_min)] = np.asarray(X_min - 1).astype(F.dtype)
        O[O < _threshold(O.dtype, X_min)] = np.asarray(X_min - 1).astype(O.dtype)
    o = O.astype(np.float64)[:, None]
    x = F.astype(np.float64)
    b1 = (x < o).sum(axis=1)
    b2 = k - (x > o).sum(axis=1)
    tied = (x == o).any(axis=1)
    counts = np.bincount(b1[~tied], minlength=k + 1).astype(np.int64)
    pairs = np.stack([b1[tied], b2[tied]], axis=1)
    if u is None:
        return counts, pairs
    assert len(u) == len(pairs)
    bins = (pairs[:, 0] + u * (pairs[:, 1] + 1 - pairs[:, 0])).astype(np.int64)
    return counts + np.bincount(bins, minlength=k + 1).astype(np.int64)


def reldiag(P_f, X_o, X_min, edges):
    P, O = np.asarray(P_f).reshape(-1), np.asarray(X_o).reshape(-1)
    keep = np.isfinite(P) & np.isfinite(O)
    P, O = P[keep], O[keep]
    edges = np.asarray(edges, dtype=np.float64)
    idx = (P.astype(np.float64)[:, None] > edges[None, :]).sum(axis=1)  # the edges below: digitize(right=True)
    event = O >= _threshold(O.dtype, X_min)
    nb = len(edges) - 1
    count = np.zeros(nb, np.int64)
    above = np.zeros(nb, np.int64)
    sums = np.zeros(nb, P.dtype)
    for b in range(1, nb + 1):
        sel = idx == b
        count[b - 1] = int(sel.sum())
        above[b - 1] = int(event[sel].sum())
        sums[b - 1] = pairwise(np.ascontiguousarray(P[sel]))
    return count, above, sums


def roc(P_f, X_o, X_min, thrs):
    P, O = np.asarray(P_f).reshape(-1), np.asarray(X_o).reshape(-1)
    keep = np.isfinite(P) & np.isfinite(O)
    P, O = P[keep].astype(np.float64), O[keep]
    event = O >= _threshold(O.dtype, X_min)
    out = np.zeros((4, len(thrs)), np.int64)
    for i, t in enumerate(np.asarray(thrs, dtype=np.float64)):
        yes = P >= t
        out[:, i] = [(yes & event).sum(), (~yes & event).sum(), (yes & ~event).sum(), (~yes & ~event).sum()]
    return tuple(out)
