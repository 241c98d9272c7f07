"""TEST INFRASTRUCTURE: a NumPy restatement of the decisions the IDW grid fill (pysteps_b200/csrc/idw.cu)
takes before it computes anything -- which kernel fills the field (idw_fill_kernel), and for every 16x16
pixel tile its search bound (tile_bound) and whether the 32-bit-key kernel keeps it (idw32_kernel's reach
test).  The arithmetic is the kernel's, operation by operation: float32 centre distances times the
float32 inverse bin width with its 1e-5 slack, the radius and the bin bound in float64, no FMA (the
library is built with --fmad=false; NumPy and Python never contract).

The tests use it to show that each case reaches the branch it claims (tiles the 32-bit keys decline,
overflow-bin tiles, tiles scanned in several unsorted rounds) and, on the host, that the bound keeps
every grid point's k nearest vectors among its tile's candidates."""
import math

import numpy as np

TX = TY = 16          # IDW_TX, IDW_TY: pixel tile of one CTA
CHUNK = 2048          # IDW_CHUNK: vectors per round, and the packed index's 11 bits
BINS = 256            # IDW_BINS: centre-distance histogram; bin 255 is the overflow bin
KEY32_LIMIT = 1 << 21  # IDW_KEY32_LIMIT: 4 * squared distance below it fits a 32-bit key
KD_SHARED_MAX = 4096  # knn_device.cuh NMAX: above it the tie recomputation builds its tree serially

NONE, KEY32, PACKED, UNPACKED, INSERT = "none", "key32", "packed", "unpacked", "insert"

_SLACK_F = np.float32(np.float32(1.0) + np.float32(1e-5))  # (1.0f + 1e-5f)


def fill_kernel(k, n, level, fastw):
    """idw_fill_kernel: the search form for k neighbours among n vectors at key level `level`."""
    if n < 1:
        return NONE
    if k != 20 or n < k:
        return INSERT
    if level == 0 or n > CHUNK:
        return UNPACKED
    return KEY32 if (level == 2 and fastw) else PACKED


def fast_weights(nvar, power, offset, mean_res):
    """fast_weights(p): dense_lucaskanade's weighting, taken by the rsqrt epilogue."""
    return nvar == 2 and power == 0.5 and mean_res == 1.0 and offset > 0.0


def key_level(xy, gx, gy):
    """coords_on_16th_grid as the host derives it (motion.lucaskanade._key_level with the grid's level):
    2 half-pixel vectors on an integer grid, 1 every coordinate a multiple of 1/16 below 2^14, else 0."""
    xy, gx, gy = (np.asarray(a, dtype=np.float64) for a in (xy, gx, gy))

    def on16(a):
        return bool(np.all(a * 16.0 == np.rint(a * 16.0)) and np.abs(a).max() < 16384.0)

    if not (on16(xy) and on16(gx) and on16(gy)):
        return 0
    ints = np.all(gx == np.rint(gx)) and np.all(gy == np.rint(gy))
    return 2 if ints and np.all(xy * 2.0 == np.rint(xy * 2.0)) else 1


class Tile:
    """tile_bound of pixel tile (bx, by): its geometry, the float32 bin of every vector, and the bound."""

    def __init__(self, xy, gx, gy, k, bx, by):
        nx, ny = len(gx), len(gy)
        self.j0, self.j1 = bx * TX, min(bx * TX + TX, nx) - 1
        self.i0, self.i1 = by * TY, min(by * TY + TY, ny) - 1
        xa, xb, ya, yb = float(gx[self.j0]), float(gx[self.j1]), float(gy[self.i0]), float(gy[self.i1])
        self.cx, self.cy = 0.5 * (xa + xb), 0.5 * (ya + yb)
        self.rt = math.sqrt(0.25 * (xb - xa) * (xb - xa) + 0.25 * (yb - ya) * (yb - ya))
        self.binw = max(self.rt, 1e-300) * 0.5
        inv_binw = 1.0 / self.binw
        with np.errstate(over="ignore", invalid="ignore"):
            inv_binw_f = np.float32(inv_binw) * _SLACK_F
            dx = (xy[:, 0] - self.cx).astype(np.float32)
            dy = (xy[:, 1] - self.cy).astype(np.float32)
            d = np.sqrt(dx * dx + dy * dy) * inv_binw_f
            # d < 255.0f ? (int)d : 255 -- NaN (0 * inf) and inf land in the overflow bin
            self.bins = np.where(d < np.float32(BINS - 1), np.where(np.isfinite(d), d, 0), BINS - 1).astype(np.int64)
        hist = np.bincount(self.bins, minlength=BINS)
        incl = np.cumsum(hist)
        reached = np.nonzero(incl >= k)[0]
        self.bk = int(reached[0]) if reached.size else BINS
        self.bmax = BINS - 1
        if self.bk < BINS - 1:
            R = (float(self.bk + 1) * self.binw + 2.0 * self.rt) * (1.0 + 1e-9)
            bb = R * inv_binw * (1.0 + 1e-9)
            self.bmax = int(bb) if bb < float(BINS - 1) else BINS - 1
        n = len(xy)
        self.total = n if self.bmax == BINS - 1 else int(incl[self.bmax])
        self.overflow = self.bmax == BINS - 1
        self.sorted = self.total <= CHUNK
        reach = 2.0 * (float(self.bmax + 1) * self.binw + self.rt) * (1.0 + 1e-6)
        self.key32 = self.sorted and not self.overflow and reach * reach < float(KEY32_LIMIT)

    def candidates(self):
        """Mask of the vectors the tile examines (all of them when it scans unsorted rounds)."""
        if not self.sorted or self.overflow:
            return np.ones(len(self.bins), dtype=bool)
        return self.bins <= self.bmax


def tiles(xy, gx, gy, k):
    """Every pixel tile's Tile, row-major (tile row by, tile column bx), for k = min(k, n) neighbours."""
    xy = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    gx, gy = np.asarray(gx, dtype=np.float64), np.asarray(gy, dtype=np.float64)
    k = min(int(k), len(xy))
    tx, ty = -(-len(gx) // TX), -(-len(gy) // TY)
    return [[Tile(xy, gx, gy, k, bx, by) for bx in range(tx)] for by in range(ty)]


def tile_bounds(xy, gx, gy, k):
    """Per tile (tile rows, tile columns): bk, bmax, total, sorted (total <= 2048) and whether the
    32-bit-key kernel keeps the tile (key32; the packed kernel behind it fills the others)."""
    ts = tiles(xy, gx, gy, k)
    return {name: np.array([[getattr(t, name) for t in row] for row in ts])
            for name in ("bk", "bmax", "total", "sorted", "key32", "overflow")}


def coverage(xy, gx, gy, k):
    """(declined by the 32-bit keys, overflow-bin, multi-round) tile counts of a fill."""
    b = tile_bounds(xy, gx, gy, k)
    return int((~b["key32"]).sum()), int(b["overflow"].sum()), int((~b["sorted"]).sum())


# ---- the geometries of the edge tests (tests/test_idw_edges_gpu.py), shared with the host checks ------
def half_points(n, x1, y1, rng, x0=0.0, y0=0.0):
    """n vectors on the half-pixel grid inside [x0, x1] x [y0, y1]."""
    return np.stack([rng.integers(int(2 * x0), int(2 * x1) + 1, n), rng.integers(int(2 * y0), int(2 * y1) + 1, n)],
                    1) / 2.0


def strip_case(n, seed=0):
    """48 x 3000 grid, n half-pixel vectors in [0, 100]^2: the 32-bit keys decline the far tiles (reach
    beyond ~724 px) and the farthest tiles' k-th bin is the overflow bin."""
    rng = np.random.default_rng(seed + n)
    return half_points(n, 100, 100, rng), np.arange(3000.0), np.arange(48.0)


def cluster_case(n, seed=0):
    """n half-pixel vectors inside 20 x 20 px on a 64 x 64 grid, an eighth of them coincident with
    others: every tile holds more than 2048 candidates and scans unsorted rounds."""
    rng = np.random.default_rng(seed + n)
    xy = half_points(n, 41.5, 41.5, rng, 22.0, 22.0)
    m = n // 8
    xy[rng.choice(n, m, replace=False)] = xy[rng.choice(n, m, replace=False)]
    return xy, np.arange(64.0), np.arange(64.0)


def partial_case(ny, nx, n=300, seed=0):
    """an ny x nx grid whose last tile row / column is partial (1 px for 17, 33, 257), vectors around it"""
    rng = np.random.default_rng(seed + 7 * ny + nx)
    return half_points(n, nx + 8, ny + 8, rng, -8.0, -8.0), np.arange(float(nx)), np.arange(float(ny))


def count_case(n, seed=0):
    """n half-pixel vectors over a 96 x 128 grid"""
    rng = np.random.default_rng(seed + n)
    return half_points(n, 127, 95, rng), np.arange(128.0), np.arange(96.0)


def mid_case(seed=0):
    """400 half-pixel vectors over a 100 x 120 grid (the k = 1 .. 32 sweep)"""
    rng = np.random.default_rng(seed + 400)
    return half_points(400, 119, 99, rng), np.arange(120.0), np.arange(100.0)


TRANSLATIONS = (0, 8000, 16383 - 63, 16384, -16384, 10 ** 6)


def translated_case(t, seed=0):
    """300 half-pixel vectors over a 48 x 64 grid, vectors and grid moved by t: from the 32-bit keys
    (t = 0) through the last level-2 offset (the grid ends at 16383) to the unpacked keys"""
    rng = np.random.default_rng(seed + 300)
    return half_points(300, 63, 47, rng) + t, np.arange(64.0) + t, np.arange(48.0) + t


def wide_case(nx, seed=0):
    """16 x nx grid with 300 half-pixel vectors along it: nx = 16383 / 16384 is the planned path's grid_ok"""
    rng = np.random.default_rng(seed + 16)
    return half_points(300, nx - 1, 15, rng), np.arange(float(nx)), np.arange(16.0)


def weight_case(seed=0):
    """300 half-pixel vectors over a 64 x 80 grid, one of them on grid point (x, y) = (10, 20)"""
    rng = np.random.default_rng(seed + 80)
    xy = half_points(300, 79, 63, rng)
    xy[5] = (10.0, 20.0)
    return xy, np.arange(80.0), np.arange(64.0)


def nonuniform_grid(n, scale):
    """geometric spacing with one value repeated: a monotonic grid of n points whose resolution differs
    from sub-grid to sub-grid"""
    g = scale * (1.05 ** np.arange(n - 1) - 1.0)
    return np.insert(g, n // 3, g[n // 3])


def nonuniform_case(seed=0):
    rng = np.random.default_rng(seed + 200)
    gx, gy = nonuniform_grid(50, 6.0), nonuniform_grid(40, 5.0)
    xy = np.stack([rng.uniform(gx[0], gx[-1], 200), rng.uniform(gy[0], gy[-1], 200)], 1)
    return xy, gx, gy


def dense_frames(seed=1):
    """two 256 x 2048 frames whose rain lies in the columns below 200: the declustered vectors sit at
    the left end of a wide grid"""
    from pysteps_b200 import _synthetic as syn
    fr = np.zeros((2, 256, 2048))
    fr[:, :, :200] = syn.rain_frames(256, 200, 2, seed)
    return fr


STRIP_NS, STRIP_KS = (300, 2048), (20, 13)
PARTIAL_GRIDS = ((17, 17), (33, 1), (1, 33), (1, 1), (255, 257))
CLUSTER_NS = (3000, 5000)
COUNT_NS = (19, 20, 21, 2047, 2048, 2049, 4096, 4097)
WIDE_NXS = (16383, 16384)


def gpu_configs():
    """(name, xy, gx, gy, ks) of every vector set the GPU edge tests fill with the tree-backed fix,
    except the dense_lucaskanade case (its vectors come from the frames)."""
    for n in STRIP_NS:
        yield (f"strip{n}",) + strip_case(n) + (STRIP_KS,)
    for ny, nx in PARTIAL_GRIDS:
        yield (f"partial{ny}x{nx}",) + partial_case(ny, nx) + ((20, 7),)
    for n in CLUSTER_NS:
        yield (f"cluster{n}",) + cluster_case(n) + ((20, 13),)
    for n in COUNT_NS:
        yield (f"count{n}",) + count_case(n) + ((20,),)
    yield ("mid",) + mid_case() + (tuple(range(1, 33)),)
    for t in TRANSLATIONS:
        yield (f"translated{t}",) + translated_case(t) + ((20,),)
    for nx in WIDE_NXS:
        yield (f"wide{nx}",) + wide_case(nx) + ((20,),)
    yield ("weights",) + weight_case() + ((20, 6),)
    yield ("nonuniform",) + nonuniform_case() + ((20,),)
