"""The edge grid of the sparse-vector cleansing of dense LK: the global and k-NN Mahalanobis outlier
tests (csrc/sparse.cu outliers_global_kernel, csrc/knn.cu + knn_body.cuh mahalanobis_outlier), the
compaction of the kept rows (compact_rows_kernel) and the per-cell medians (decluster_kernel).

Every case names the kernel branches it is there for; `classify` works those branches out from the
case's shape, contents and arguments alone, and the coverage test of tests/test_oracle_sparse_edges.py
holds the names to it.  `md_extended` is the reference's Mahalanobis distance in extended precision, so
that decisions within rounding of the threshold (`MD_MARGIN`) can be told apart from real differences.

tests/test_oracle_sparse_edges.py pins the oracle to the reference on this grid (CPU);
tests/test_sparse_edges_gpu.py holds the device to the oracle on it."""
import functools

import numpy as np

NBSMEM = 32        # csrc/knn_device.cuh: k + 1 <= NBSMEM takes the warp query
NMAX = 4096        # csrc/knn_device.cuh: n_cap <= NMAX takes the shared-memory tree build
QHEAP = 64         # csrc/knn_device.cuh: pending-node heap of one query
ARENA = 1 << 17    # csrc/knn_device.cuh: spill entries of one call
DC_MAX = 16384     # csrc/sparse.cu
DC_BIAS = 1 << 24  # csrc/sparse.cu: finite cells in [1 - DC_BIAS, DC_BIAS - 2]
MD_MARGIN = 1e-9   # relative: |MD - thr| <= MD_MARGIN * max(1, cond(V)) * max(1, thr) is a tie

# ------------------------------------------------------------------------------------------ data
def _uv(n, rng, spikes=7):
    """dyadic (1/256) vectors around (2, -1) with a spike every `spikes` rows: sums of a few hundred of
    them are exact, so singular neighbour sets are singular in every summation order"""
    uv = np.stack([2 + rng.integers(-96, 97, n) / 256.0, -1 + rng.integers(-96, 97, n) / 256.0], 1)
    if spikes:
        uv[::spikes] += rng.integers(-3, 4, (len(uv[::spikes]), 2)) * 0.5
    return uv


def _coords(kind, n, rng):
    if kind == "lattice":
        side = int(np.ceil(np.sqrt(max(n, 1))))
        g = np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2)[:n]
        return g[rng.permutation(n)].astype(np.float64) * 3.0
    if kind == "coincident":
        base = rng.integers(0, max(4, int(np.sqrt(n) * 2)), (max(n // 3, 1), 2)).astype(np.float64)
        return base[rng.integers(0, len(base), n)]
    if kind == "half":
        return rng.integers(0, 2 * max(8, int(np.sqrt(n) * 3)), (n, 2)) / 2.0
    if kind == "constx":
        xy = rng.integers(0, 5 * n + 5, (n, 2)).astype(np.float64)
        xy[:, 0] = 11.0
        return xy
    raise KeyError(kind)


# ---------------------------------------------------------------------- global outlier test
def _global_uv(kind, n, rng):
    if kind == "random":
        return _uv(n, rng)
    if kind == "swap":     # |cov(u, v)| > var(u): the LU pivots on the second row
        t = rng.integers(-64, 65, n) / 64.0
        return np.stack([t + rng.integers(-4, 5, n) / 256.0, 3 * t + rng.integers(-8, 9, n) / 64.0], 1)
    if kind == "ucon":     # u constant: var(u) = cov = 0, p0 == 0
        return np.stack([np.full(n, 1.25), rng.integers(-64, 65, n) / 64.0], 1)
    if kind == "vcon":     # v constant: cov = var(v) = 0, u22 == 0
        return np.stack([rng.integers(-64, 65, n) / 64.0, np.full(n, -0.5)], 1)
    if kind == "collinear":
        # v = 2u, u symmetric about 0 and n - 1 a power of two: V = [[1, 2], [2, 4]] exactly in any
        # order of summation; both LUs pivot on 2 and find u22 = 2 - 0.5 * 4 = 0
        assert n - 1 & n - 2 == 0 and n % 2 == 1
        h = (n - 1) // 2
        t = np.concatenate([np.ones(h), -np.ones(h), [0.0]])[rng.permutation(n)]
        return np.stack([t * np.sqrt((n - 1) / (2.0 * h)), 2 * t * np.sqrt((n - 1) / (2.0 * h))], 1)
    raise KeyError(kind)


def _g(name, n, kind="random", thr=2.0, n_dev=None, claims=()):
    return name, dict(op="global", n=n, kind=kind, thr=thr, n_dev=n_dev, claims=tuple(claims))


# n: the rows that count; n_dev: None (the count is n_cap = n) or the device count (n_cap = n + pad
# rows of garbage, or fewer rows than n_dev: clamped)
GLOBAL = dict([
    _g("g-n0", 0, n_dev=0, claims=["g:n<2", "g:ndev<cap"]),
    _g("g-n1", 1, n_dev=1, claims=["g:n<2"]),
    _g("g-n2", 2, claims=["g:n=2"]),
    _g("g-n255", 255, claims=["g:n=255"]),
    _g("g-n256", 256, thr=1.5, claims=["g:n=256"]),
    _g("g-n257", 257, claims=["g:n=257", "g:keep"]),
    _g("g-n3000-ndev", 3000, thr=2.5, n_dev=3000, claims=["g:strides", "g:ndev<cap"]),
    _g("g-n700-clamped", 700, n_dev=900, claims=["g:ndev>cap"]),
    _g("g-swap", 1000, "swap", 2.0, claims=["g:swap"]),
    _g("g-ucon", 300, "ucon", 1.0, claims=["g:p0=0"]),
    _g("g-vcon", 300, "vcon", 1.0, claims=["g:u22=0"]),
    _g("g-collinear", 257, "collinear", 0.5, claims=["g:collinear"]),
    _g("g-collinear-ndev", 17, "collinear", 0.5, n_dev=17, claims=["g:collinear"]),
])


def global_lu(uv):
    """The LU branch both sides take on the reference's V (np.cov of the exact data)."""
    if len(uv) < 2:
        return "n<2"
    V = np.cov((uv - uv.mean(0)).T)
    a, b, d = V[0, 0], V[0, 1], V[1, 1]
    swap = abs(b) > abs(a)
    p0, p1, q0, q1 = (b, d, a, b) if swap else (a, b, b, d)
    if p0 == 0 or np.isnan(p0):
        return "p0=0"
    l = q0 * (1.0 / p0)
    if q1 - l * p1 == 0:
        return "collinear" if swap and a != 0 else "u22=0"
    return "swap" if swap else "keep"


# ------------------------------------------------------------------------- k-NN outlier test
def _k(name, n, kind, k, thr=2.0, n_dev=None, special=None, claims=()):
    return name, dict(op="knn", n=n, kind=kind, k=k, thr=thr, n_dev=n_dev, special=special, claims=tuple(claims))


KNN = dict([
    _k("k-lattice1500-k30", 1500, "lattice", 30, claims=["k:shared", "k:warp30", "k:lattice"]),
    _k("k-coinc4096-k31", 4096, "coincident", 31, claims=["k:warp31", "k:coincident"]),
    _k("k-half3000-k32-ndev", 3000, "half", 32, n_dev=4096, claims=["k:shared+ndev", "k:thread32", "k:half"]),
    _k("k-constx2000-k100", 2000, "constx", 100, 2.5, claims=["k:thread100", "k:constcoord"]),
    _k("k-half4097-k30", 4097, "half", 30, claims=["k:serial"]),
    _k("k-lattice16000-k31", 16000, "lattice", 31, claims=["k:serial"]),
    _k("k-coinc6000-k32-ndev", 6000, "coincident", 32, n_dev=6500, claims=["k:serial+ndev"]),
    _k("k-lattice5000-k100-ndev", 5000, "lattice", 100, 3.0, n_dev=5000, claims=["k:serial+ndev", "k:thread100"]),
    _k("k-n0", 0, "lattice", 30, n_dev=0, claims=["k:n<2"]),
    _k("k-n1", 1, "lattice", 30, n_dev=1, claims=["k:n<2"]),
    _k("k-n2", 2, "half", 30, claims=["k:m=1", "k:kk=n"]),
    _k("k-n2-k100", 2, "lattice", 100, claims=["k:m=1"]),
    _k("k-n5-k32", 5, "coincident", 32, 1.0, claims=["k:kk=n"]),
    _k("k-n31-k30", 31, "lattice", 30, 1.0, claims=["k:kk=n"]),
    _k("k-n40-k100", 40, "half", 100, 1.0, claims=["k:kk=n"]),
    _k("k-identical-uv", 1200, "coincident", 30, special="identical", claims=["k:sing_identical"]),
    _k("k-constv", 1200, "lattice", 31, special="constv", claims=["k:sing_constv"]),
    _k("k-constv-k32", 900, "half", 32, special="constv", claims=["k:sing_constv", "k:thread32"]),
])


# --------------------------------------------------------------------------------- compaction
def _c(name, n, pattern, n_dev=None, claims=()):
    return name, dict(op="compact", n=n, pattern=pattern, n_dev=n_dev, claims=tuple(claims))


COMPACT = dict([
    _c("c-n0", 0, "random", n_dev=0, claims=["c:n=0"]),
    _c("c-n1", 1, "none", claims=["c:n=1"]),
    _c("c-n31", 31, "alternate", claims=["c:n=31", "c:partial_warp"]),
    _c("c-n32", 32, "all", claims=["c:n=32", "c:all_dropped"]),
    _c("c-n1023", 1023, "random", claims=["c:n=1023"]),
    _c("c-n1024", 1024, "none", claims=["c:n=1024", "c:none_dropped"]),
    _c("c-n1025", 1025, "alternate", claims=["c:n=1025", "c:alternating", "c:rounds>1"]),
    _c("c-n5000", 5000, "random", claims=["c:n=5000"]),
    _c("c-n5000-ndev", 5000, "random", n_dev=5000, claims=["c:ndev", "c:n=5000"]),
    _c("c-n3000-clamped", 3000, "alternate", n_dev=3500, claims=["c:ndev"]),
])


def compact_drop(c, rng):
    n = c["n"]
    if c["pattern"] == "none":
        return np.zeros(n, np.uint8)
    if c["pattern"] == "all":
        return np.ones(n, np.uint8)
    if c["pattern"] == "alternate":
        return (np.arange(n) % 2).astype(np.uint8)
    return (rng.random(n) < 0.3).astype(np.uint8)


# ---------------------------------------------------------------------------------- decluster
def _d(name, n, kind, scale=20.0, min_samples=1, claims=()):
    return name, dict(op="decluster", n=n, kind=kind, scale=scale, min_samples=min_samples, claims=tuple(claims))


DECLUSTER = dict([
    _d("d-n1", 1, "frame", claims=["d:n=1"]),
    _d("d-n2-even", 2, "onecell", claims=["d:n=2", "d:even"]),
    _d("d-n1024", 1024, "frame", claims=["d:n=1024", "d:min1"]),
    _d("d-n1025", 1025, "frame", claims=["d:per>1"]),
    _d("d-n4096-ms2", 4096, "ties", 20.0, 2, claims=["d:n=4096", "d:min2", "d:tie"]),
    _d("d-n16384-own", DC_MAX, "own", 1.0, claims=["d:DC_MAX", "d:own_cells"]),
    _d("d-n16384-ms3", DC_MAX, "frame", 7.5, 3, claims=["d:DC_MAX", "d:nonint_scale"]),
    _d("d-onecell-odd", 2999, "onecell", claims=["d:one_cell", "d:odd"]),
    _d("d-onecell-even", 2000, "onecell", 1000.0, claims=["d:one_cell", "d:even"]),
    _d("d-negative", 3000, "negative", 7.0, claims=["d:negative"]),
    _d("d-edges", 800, "edges", 20.0, claims=["d:edge"]),
    _d("d-roundedge", 400, "roundedge", 0.1, claims=["d:round_edge", "d:nonint_scale"]),
    _d("d-ms0", 500, "frame", 20.0, 0, claims=["d:min0"]),
    _d("d-ms-gt-n", 300, "frame", 20.0, 301, claims=["d:min>n"]),
    _d("d-near2^20", 600, "near2^20", 1.0, claims=["d:near2^20"]),
    _d("d-beyond2^20", 600, "beyond2^20", 1.0, claims=["d:beyond2^20"]),
    _d("d-near2^24", 600, "near2^24", 1.0, claims=["d:near2^24"]),
    _d("d-beyond2^24", 600, "beyond2^24", 1.0, claims=["d:refused_range"]),
    _d("d-nonfinite", 500, "nonfinite", 20.0, claims=["d:nan", "d:inf"]),
    _d("d-nonfinite-ms2", 500, "nonfinite", 20.0, 2, claims=["d:nan"]),
    _d("d-nan-ms0", 500, "nonfinite", 20.0, 0, claims=["d:refused_nan"]),
])
DC_OVER = DC_MAX + 1  # refused with B200_ENOTSUP


def decluster_inputs(c):
    """(coord, values) of a decluster case"""
    n, kind = c["n"], c["kind"]
    rng = np.random.default_rng(n * 31 + len(kind))
    uv = np.stack([rng.integers(-512, 513, n) / 128.0, rng.integers(-512, 513, n) / 128.0], 1)
    if kind == "frame":
        xy = rng.integers(0, 1024, (n, 2)).astype(np.float64)
    elif kind == "onecell":
        xy = rng.integers(0, int(c["scale"]), (n, 2)) + rng.integers(0, 4, (n, 2)) / 4.0
    elif kind == "ties":   # few distinct values: equal values inside most cells
        xy = rng.integers(0, 160, (n, 2)).astype(np.float64)
        uv = rng.integers(-2, 3, (n, 2)) / 2.0
    elif kind == "own":    # 128 x 128 cells of side 1, one point each, shuffled
        g = np.stack(np.meshgrid(np.arange(128), np.arange(128)), -1).reshape(-1, 2)[rng.permutation(n)]
        xy = g + 0.5
    elif kind == "negative":
        xy = rng.integers(-300, 300, (n, 2)) + rng.integers(0, 2, (n, 2)) * 0.5
    elif kind == "edges":  # on the edges k * scale and just either side of them
        e = rng.integers(-10, 10, (n, 2)) * c["scale"]
        xy = e + rng.choice([0.0, -1e-9, 1e-9, -0.5, 0.5], (n, 2))
    elif kind == "roundedge":  # 0.3 / 0.1 = 2.9999999999999996: cell 2, not 3
        xy = rng.choice([0.1, 0.2, 0.3, 0.6, 0.7, 1.1, 2.3, -0.3, -0.7, 0.30000000000000004], (n, 2))
    elif kind in ("near2^20", "beyond2^20", "near2^24", "beyond2^24"):
        e = {"near2^20": 2 ** 20, "beyond2^20": 2 ** 20 + 902848, "near2^24": DC_BIAS, "beyond2^24": DC_BIAS}[kind]
        lo, hi = {"near2^24": (1 - e, e - 2), "beyond2^24": (-e, e - 1)}.get(kind, (-e - 3, e + 3))
        xy = rng.choice([lo, lo + 1.0, hi - 1.0, hi, 0.0, hi - 902848.0], (n, 2)) + rng.integers(0, 4, (n, 2)) / 4.0
        if kind == "beyond2^20":  # x = 3e6 and x = 902848 share the old 21-bit key
            xy[:2, 0] = [3e6, 902848.0]
    elif kind == "nonfinite":
        xy = rng.integers(-60, 60, (n, 2)).astype(np.float64)
        for j, v in enumerate((np.nan, np.inf, -np.inf)):
            xy[j::7, j % 2] = v
        xy[5::11] = np.inf
    else:
        raise KeyError(kind)
    return np.ascontiguousarray(xy, dtype=np.float64), np.ascontiguousarray(uv)


def decluster_vectorised(coord, values, scale, min_samples=1):
    """cleansing.py:21-121 restated with one lexsort and a per-cell median (O(n log n)): the oracle's
    loop over cells is O(n * cells).  Rows with a NaN cell belong to no cell; min_samples < 1 with NaN
    rows (the reference then appends NaN medians) is not restated."""
    cells = np.floor(coord / float(scale)) + 0.0  # -0.0 -> 0.0: np.unique compares them equal
    ok = ~np.isnan(cells).any(1)
    assert ok.all() or min_samples >= 1
    idx = np.nonzero(ok)[0]
    idx = idx[np.lexsort((cells[idx, 1], cells[idx, 0]))]
    cs = cells[idx]
    head = np.ones(len(idx), bool)
    head[1:] = (cs[1:] != cs[:-1]).any(1)
    starts = np.nonzero(head)[0]
    ends = np.append(starts[1:], len(idx))
    oxy, ouv = [], []
    for s, e in zip(starts, ends):
        if e - s >= min_samples:
            oxy.append(np.median(coord[idx[s:e]], axis=0))
            ouv.append(np.median(values[idx[s:e]], axis=0))
    return np.array(oxy).reshape(-1, 2), np.array(ouv).reshape(-1, 2)


def decluster_refused(coord, scale, min_samples):
    """The kernel refuses (out_count = -1): a finite cell beyond its key, or NaN rows with min_samples < 1"""
    with np.errstate(all="ignore"):
        cells = np.floor(coord / float(scale))
    fin = cells[np.isfinite(cells)]
    return bool(np.any((fin < 1 - DC_BIAS) | (fin > DC_BIAS - 2)) or (np.isnan(cells).any() and min_samples < 1))


# --------------------------------------------------------------------------------- case inputs
@functools.lru_cache(maxsize=None)
def knn_inputs(tag):
    """(xy, uv) of a k-NN case: n rows that count"""
    c = KNN[tag]
    n = c["n"]
    rng = np.random.default_rng(1000 + n + c["k"] + len(c["kind"]))
    xy, uv = _coords(c["kind"], n, rng), _uv(n, rng)
    if c["special"] == "identical" and n:
        # a block of 200 rows (a whole region of the set) with one vector: their neighbour sets
        # are that vector alone
        region = np.argsort(xy[:, 0] + 1e-3 * xy[:, 1], kind="stable")[:200]
        uv[region] = (1.5, -0.75)
    elif c["special"] == "constv" and n:
        region = np.argsort(xy[:, 1] + 1e-3 * xy[:, 0], kind="stable")[:300]
        uv[region, 1] = -0.25
    return np.ascontiguousarray(xy), np.ascontiguousarray(uv)


@functools.lru_cache(maxsize=None)
def global_inputs(tag):
    c = GLOBAL[tag]
    rng = np.random.default_rng(77 + c["n"] + len(c["kind"]))
    return np.ascontiguousarray(_global_uv(c["kind"], c["n"], rng) if c["n"] else np.zeros((0, 2)))


PAD = 37  # garbage rows past the count when the count is on the device


def n_cap(c):
    """the capacity the entry point is called with: n_dev == n leaves PAD garbage rows past the count,
    n_dev > n is clamped to the capacity n"""
    if c["n_dev"] is None or c["n_dev"] > c["n"]:
        return c["n"]
    assert c["n_dev"] == c["n"]
    return c["n"] + PAD


def device_count(c):
    """min(*n_dev, n_cap): the rows that count on the device"""
    return c["n"]


# --------------------------------------------------------------------------------- the classifier
def knn_neighbours(xy, k):
    """cKDTree's neighbour lists (oracle/ckdtree.py, pinned to scipy) of every row, kk = min(k + 1, n)"""
    from oracle.ckdtree import KDTree
    n = len(xy)
    kk = min(k + 1, n)
    _, inds = KDTree(xy).query(xy, k=kk)
    return np.asarray(inds).reshape(n, kk)


def _cov_parts(nb):
    """a, b, d of np.cov over the last-but-one axis (extended precision), nb (..., m, 2)"""
    mu = nb.mean(axis=-2, keepdims=True)
    z = nb - mu
    z = z - z.mean(axis=-2, keepdims=True)
    m = nb.shape[-2]
    f = np.longdouble(1) / np.longdouble(m - 1) if m > 1 else np.longdouble(np.inf)
    with np.errstate(all="ignore"):
        return ((z[..., 0] ** 2).sum(-1) * f, (z[..., 0] * z[..., 1]).sum(-1) * f, (z[..., 1] ** 2).sum(-1) * f, mu[..., 0, :])


def md_extended(uv, inds=None):
    """(MD, singular, cond) of every row in extended precision: the reference's distance of uv[i] to the
    mean of its neighbours inds[i, 1:] (all rows when inds is None, the global test) under their sample
    covariance.  Singular (or m = 1) rows have MD 0, as the reference's LinAlgError branch gives."""
    U = uv.astype(np.longdouble)
    if inds is None:
        nb = U[None]
        a, b, d, mu = _cov_parts(nb)
        z = U - mu
    else:
        nb = U[inds[:, 1:]]
        a, b, d, mu = _cov_parts(nb)
        z = U - mu
    with np.errstate(all="ignore"):
        det = a * d - b * b
        sing = ~(det != 0) | ~np.isfinite(det)
        q = (z[:, 0] ** 2 * d - 2 * z[:, 0] * z[:, 1] * b + z[:, 1] ** 2 * a) / det
        md = np.where(sing, 0, np.sqrt(np.abs(q)))
        tr = a + d
        disc = np.sqrt(np.maximum((a - d) ** 2 + 4 * b * b, 0))
        cond = np.where(sing, np.inf, (tr + disc) / np.maximum(tr - disc, 1e-300))
    return md.astype(np.float64), np.broadcast_to(sing, md.shape), np.broadcast_to(cond, md.shape).astype(np.float64)


def tie_rows(md, sing, cond, thr):
    """rows whose decision may legitimately differ between two float64 summation orders"""
    margin = MD_MARGIN * np.maximum(1.0, cond) * max(1.0, thr)
    return ~sing & (np.abs(md - thr) <= margin)


def classify(tag):
    """the branches a case takes, worked out from its inputs and arguments"""
    for table in (GLOBAL, KNN, COMPACT, DECLUSTER):
        if tag in table:
            c = table[tag]
            break
    else:
        raise KeyError(tag)
    op, out = c["op"], set()
    if op == "global":
        n, cap = device_count(c), n_cap(c)
        uv = global_inputs(tag)[:n]
        if n < 2:
            out.add("g:n<2")
        if n in (2, 255, 256, 257):
            out.add(f"g:n={n}")
        if n > 2 * 256:
            out.add("g:strides")
        if c["n_dev"] is not None:
            out.add("g:ndev<cap" if c["n_dev"] < cap else "g:ndev>cap" if c["n_dev"] > cap else "g:ndev=cap")
        out.add("g:" + global_lu(uv))
    elif op == "knn":
        n, cap, k = device_count(c), n_cap(c), c["k"]
        xy, uv = knn_inputs(tag)
        build = "shared" if cap <= NMAX else "serial"
        out.add(f"k:{build}" + ("+ndev" if c["n_dev"] is not None and n >= 2 else ""))
        if n < 2:
            out.add("k:n<2")
            return out
        out.add(f"k:warp{k}" if k + 1 <= NBSMEM else f"k:thread{k}")
        if min(k + 1, n) == n:
            out.add("k:kk=n")
        if n == 2:
            out.add("k:m=1")
        if np.ptp(xy[:, 0]) == 0 or np.ptp(xy[:, 1]) == 0:
            out.add("k:constcoord")
        elif np.any(xy != np.floor(xy)):
            out.add("k:half")
        elif len(np.unique(xy, axis=0)) < n:
            out.add("k:coincident")
        else:
            out.add("k:lattice")
        inds = knn_neighbours(xy, k)
        a, b, d, _ = _cov_parts(uv.astype(np.longdouble)[inds[:, 1:]])
        if np.any((a == 0) & (b == 0) & (d == 0)):
            out.add("k:sing_identical")
        if np.any((d == 0) & (a > 0)):
            out.add("k:sing_constv")
    elif op == "compact":
        n = device_count(c)
        for v in (0, 1, 31, 32, 1023, 1024, 1025, 5000):
            if n == v:
                out.add(f"c:n={v}")
        if n > 1024:
            out.add("c:rounds>1")
        if n % 32:
            out.add("c:partial_warp")
        if c["n_dev"] is not None:
            out.add("c:ndev")
        drop = compact_drop(c, np.random.default_rng(0))[:n]
        if n:
            out.add("c:none_dropped" if not drop.any() else "c:all_dropped" if drop.all() else
                    "c:alternating" if np.array_equal(drop, np.arange(n) % 2) else "c:some_dropped")
    else:
        xy, uv = decluster_inputs(c)
        n, scale, ms = c["n"], float(c["scale"]), c["min_samples"]
        for v, name in ((1, "n=1"), (2, "n=2"), (1024, "n=1024"), (4096, "n=4096"), (DC_MAX, "DC_MAX")):
            if n == v:
                out.add("d:" + name)
        npad = 1 << max(1, int(np.ceil(np.log2(max(n, 2)))))
        if -(-npad // 1024) > 1:
            out.add("d:per>1")
        if scale != np.floor(scale):
            out.add("d:nonint_scale")
        with np.errstate(all="ignore"):
            cells = np.floor(xy / scale)
        if np.isnan(cells).any():
            out.add("d:nan")
        if np.isinf(cells).any():
            out.add("d:inf")
        if decluster_refused(xy, scale, ms):
            out.add("d:refused_nan" if np.isnan(cells).any() and ms < 1 else "d:refused_range")
            return out
        fin = cells[np.isfinite(cells)]
        if fin.size and np.abs(fin).max() >= 2 ** 20 - 4 and np.abs(fin).max() < 2 ** 20 + 4:
            out.add("d:near2^20")
        if fin.size and np.abs(fin).max() >= 2 ** 20 + 4 and np.abs(fin).max() < DC_BIAS - 4:
            out.add("d:beyond2^20")
        if fin.size and np.abs(fin).max() >= DC_BIAS - 4:
            out.add("d:near2^24")
        if (xy < 0).any():
            out.add("d:negative")
        if np.any(xy[np.isfinite(xy)] == np.floor(xy[np.isfinite(xy)] / scale) * scale):
            out.add("d:edge")
        with np.errstate(all="ignore"):
            q = xy / scale
            if np.any(np.isfinite(q) & (np.floor(q) != np.floor(np.round(q, 9))) & (np.abs(q - np.round(q)) < 1e-9)):
                out.add("d:round_edge")
        ok = ~np.isnan(cells).any(1)
        _, counts = np.unique(cells[ok] + 0.0, axis=0, return_counts=True)
        if counts.size and counts.max() == 1:
            out.add("d:own_cells")
        if len(counts) == 1:
            out.add("d:one_cell")
        if np.any(counts % 2 == 1):
            out.add("d:odd")
        if np.any(counts % 2 == 0):
            out.add("d:even")
        if ms in (0, 1, 2):
            out.add(f"d:min{ms}")
        elif ms > n:
            out.add("d:min>n")
        # equal values inside a cell of at least three (the rank tie q < p decides the median)
        cid = np.unique(cells[ok] + 0.0, axis=0, return_inverse=True)[1].ravel()
        vals = uv[ok]
        key = np.stack([cid, vals[:, 0]], 1)
        if len(np.unique(key, axis=0)) < len(key):
            out.add("d:tie")
    return out


BRANCHES = {
    "global": ["g:n<2", "g:n=2", "g:n=255", "g:n=256", "g:n=257", "g:strides", "g:ndev<cap", "g:ndev>cap",
               "g:keep", "g:swap", "g:p0=0", "g:u22=0", "g:collinear"],
    "knn": ["k:shared", "k:serial", "k:shared+ndev", "k:serial+ndev", "k:warp30", "k:warp31", "k:thread32",
            "k:thread100", "k:kk=n", "k:m=1", "k:n<2", "k:lattice", "k:coincident", "k:half", "k:constcoord",
            "k:sing_identical", "k:sing_constv"],
    "compact": ["c:n=0", "c:n=1", "c:n=31", "c:n=32", "c:n=1023", "c:n=1024", "c:n=1025", "c:n=5000",
                "c:rounds>1", "c:none_dropped", "c:all_dropped", "c:alternating", "c:partial_warp", "c:ndev"],
    "decluster": ["d:n=1", "d:n=2", "d:n=1024", "d:per>1", "d:n=4096", "d:DC_MAX", "d:own_cells", "d:one_cell",
                  "d:odd", "d:even", "d:tie", "d:negative", "d:edge", "d:round_edge", "d:nonint_scale",
                  "d:min0", "d:min1", "d:min2", "d:min>n", "d:near2^20", "d:beyond2^20", "d:near2^24",
                  "d:refused_range", "d:nan", "d:inf", "d:refused_nan"],
}
ALL_CASES = {**GLOBAL, **KNN, **COMPACT, **DECLUSTER}
