"""CPU oracle of the constant advection method (pysteps/motion/constant.py:20-54), restated in the
order of csrc/constant.cu so that every device evaluation can be compared with it bit for bit:

  * the tap of ``map_coordinates(prev, [Y + vy, X + vx], order=0, mode="constant", cval=nan)``:
    outside [0, m-1] x [0, n-1] -> nan, else prev[floor(y + vy + 0.5), floor(x + vx + 0.5)] + 0.0
  * the means: NumPy's pairwise summation (np.add.reduce seeded with 0.0; leaves of <= 128 values
    summed with 8 accumulators; a node of n > 128 values splits after n / 2 rounded down to a
    multiple of 8), divided by N -- equal to np.mean bit for bit
  * S00, S11, S01: lane i % 65536 sums its ranks in sequence, a halving tree over each 256 lanes,
    then the 256 CTA sums in sequence (the reference's BLAS order cannot be matched)
  * corrcoef's tail in NumPy's order, with the floating-point events as B200_CONST_* bits
"""
import numpy as np
import scipy.optimize as op

LEAF = 128
SUM_BLOCKS, SUM_THREADS = 256, 256

EMPTY, DOF, SCALE_INVALID = 1, 2, 4
ROW_INVALID, ROW_DIVZERO, ROW_OVERFLOW = 8, 16, 32
COL_INVALID, COL_DIVZERO, COL_OVERFLOW = 64, 128, 256

_leaf_cache = {}


def _leaves(n):
    """(offset, size) of the leaves of the pairwise tree over n values, left to right."""
    hit = _leaf_cache.get(n)
    if hit is not None:
        return hit
    if n <= LEAF:
        out = ((0, n),)
    else:
        h = (n // 2) - (n // 2) % 8
        out = _leaves(h) + tuple((o + h, s) for o, s in _leaves(n - h))
    if len(_leaf_cache) < 4096:
        _leaf_cache[n] = out
    return out


def _leaf_sums(a, leaves):
    """numpy's pairwise_sum of every leaf (vectorised over the leaves of one size)."""
    out = np.empty(len(leaves))
    offs = np.array([o for o, _ in leaves], dtype=np.int64)
    sizes = np.array([s for _, s in leaves], dtype=np.int64)
    for s in np.unique(sizes):
        sel = np.nonzero(sizes == s)[0]
        M = a[offs[sel, None] + np.arange(s)[None, :]]
        if s < 8:
            res = np.zeros(len(sel))
            for i in range(s):
                res = res + M[:, i]
        else:
            r = M[:, :8].copy()
            i = 8
            while i < s - s % 8:
                r = r + M[:, i:i + 8]
                i += 8
            res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
            while i < s:
                res = res + M[:, i]
                i += 1
        out[sel] = res
    return out


def pairwise_sum(a):
    """np.add.reduce(a) of a float64 vector, restated: the leaves, then the tree (left + right)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    n = a.size
    leaves = _leaves(n)
    sums = iter(_leaf_sums(a, leaves).tolist())

    def node(size):
        if size <= LEAF:
            return next(sums)
        h = (size // 2) - (size // 2) % 8
        left = node(h)
        return left + node(size - h)

    return 0.0 + node(n)


def mean(a):
    """np.mean of a float64 vector (nan for an empty one, without a warning)."""
    with np.errstate(invalid="ignore"):
        return float(np.float64(pairwise_sum(a)) / np.float64(len(a)))


def counted_values(prev, nxt, vx, vy):
    """(next[mask], warped[mask]) as float64, raster order."""
    m, n = nxt.shape
    nx = np.asarray(nxt, dtype=np.float64)
    cy = np.arange(m, dtype=np.float64)[:, None] + vy
    cx = np.arange(n, dtype=np.float64)[None, :] + vx
    inside = (cy >= 0.0) & (cy <= m - 1) & (cx >= 0.0) & (cx <= n - 1)
    with np.errstate(invalid="ignore"):
        iy = np.clip(np.floor(cy + 0.5), 0, max(m - 1, 0)).astype(np.int64)
        ix = np.clip(np.floor(cx + 0.5), 0, max(n - 1, 0)).astype(np.int64)
    warped = np.full((m, n), np.nan)
    if m and n:
        w = 0.0 + np.asarray(prev, dtype=np.float64)[iy, ix]
        warped = np.where(inside, w, np.nan)
    mask = np.isfinite(nx) & np.isfinite(warped)
    return nx[mask], warped[mask]


def centred_sums(a, b, ma, mb):
    """S00, S11, S01 in the device order."""
    N = a.size
    lanes = SUM_BLOCKS * SUM_THREADS
    rows = -(-N // lanes)
    acc = np.zeros((3, lanes))
    if N:
        xa, xb = a - ma, b - mb
        prods = [xa * xa, xb * xb, xa * xb]
        for k in range(3):
            p = np.zeros(rows * lanes)
            p[:N] = prods[k]  # a padded +0.0 leaves a lane's sum (never -0.0) unchanged
            p = p.reshape(rows, lanes)
            for r in range(rows):
                acc[k] = acc[k] + p[r]
    v = acc.reshape(3, SUM_BLOCKS, SUM_THREADS)
    s = SUM_THREADS // 2
    while s > 0:
        v[:, :, :s] = v[:, :, :s] + v[:, :, s:2 * s]
        s //= 2
    out = []
    for k in range(3):
        t = 0.0
        for g in range(SUM_BLOCKS):
            t += float(v[k, g, 0])
        out.append(t)
    return out


def _quotient_events(x, y, invalid, divzero, overflow):
    if np.isnan(x) or np.isnan(y):
        return 0
    if (x == 0.0 and y == 0.0) or (np.isinf(x) and np.isinf(y)):
        return invalid
    if y == 0.0:
        return 0 if np.isinf(x) else divzero
    with np.errstate(all="ignore"):
        if np.isfinite(x) and np.isinf(np.float64(x) / np.float64(y)):
            return overflow
    return 0


def tail(S00, S11, S01, N):
    """-> (f, flags): corrcoef after the dot product, in NumPy's order."""
    flags = EMPTY if N == 0 else 0
    fact = float(N - 1)
    if N - 1 <= 0:
        flags |= DOF
        fact = 0.0
    with np.errstate(all="ignore"):
        inv = np.float64(1.0) / np.float64(fact)
        c = np.array([[S00, S01], [S01, S11]], dtype=np.float64)
        if np.any(((c == 0.0) & np.isinf(inv)) | (np.isinf(c) & (inv == 0.0))):
            flags |= SCALE_INVALID
        c = c * inv
        sd = np.sqrt(np.diag(c).copy())
        for i in range(2):
            for j in range(2):
                flags |= _quotient_events(c[i, j], sd[i], ROW_INVALID, ROW_DIVZERO, ROW_OVERFLOW)
        c = c / sd[:, None]
        for i in range(2):
            for j in range(2):
                flags |= _quotient_events(c[i, j], sd[j], COL_INVALID, COL_DIVZERO, COL_OVERFLOW)
        c = c / sd[None, :]
    r = float(c[0, 1])
    r = -1.0 if r < -1.0 else (1.0 if r > 1.0 else r)
    return -r, flags


def evaluate(prev, nxt, vx, vy):
    """One evaluation of the objective: (f, N, flags), as b200_constant_eval."""
    a, b = counted_values(prev, nxt, float(vx), float(vy))
    N = a.size
    ma, mb = mean(a), mean(b)
    S00, S11, S01 = centred_sums(a, b, ma, mb)
    f, flags = tail(S00, S11, S01, N)
    return f, N, flags


def minimize(R):
    """scipy's Nelder-Mead on the oracle objective, with the reference's arguments (constant.py:51-52)."""
    R = np.ma.getdata(R)
    prev, nxt = R[-2], R[-1]
    options = {"initial_simplex": (np.array([(0, 1), (1, 0), (1, 1)]))}
    return op.minimize(lambda v: evaluate(prev, nxt, v[0], v[1])[0], (1, 1), method="Nelder-Mead", options=options)


def constant(R):
    """The reference's returned field, from the oracle objective."""
    m, n = R.shape[1:]
    x = minimize(R).x
    return np.stack([-x[0] * np.ones((m, n)), -x[1] * np.ones((m, n))])
