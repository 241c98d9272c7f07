"""Host checks of the IDW grid fill's tile search (pysteps_b200/csrc/idw.cu), through its restatement in
idw_tiles.py: the per-tile search bound keeps every grid point's k nearest vectors (and any vector tied
with the k-th) among the tile's candidates, the 32-bit keys the kernel accepts fit in 32 bits, the
packed 64-bit keys leave their 11 index bits free at the extremes of level 1, and the tree queries of
the tie recomputation never outgrow their 64-entry heap on the GPU edge tests' vector sets."""
import ctypes

import numpy as np
import pytest

import idw_tiles as T


def _grid_d2(xy, gx, gy, i0, i1, j0, j1, sel=None):
    """Exact squared distances (in 1/256 px^2) of the grid points [i0..i1] x [j0..j1] to the vectors
    (all, or the masked ones): every coordinate here is a multiple of 1/16."""
    pts = xy if sel is None else xy[sel]
    X, Y = np.rint(pts[:, 0] * 16).astype(np.int64), np.rint(pts[:, 1] * 16).astype(np.int64)
    qx = np.rint(gx[j0:j1 + 1] * 16).astype(np.int64)
    qy = np.rint(gy[i0:i1 + 1] * 16).astype(np.int64)
    QX, QY = np.meshgrid(qx, qy)
    dx, dy = X[None, :] - QX.reshape(-1, 1), Y[None, :] - QY.reshape(-1, 1)
    return dx * dx + dy * dy


def _check_bound(xy, gx, gy, k):
    """Every grid point: all vectors at most as far as its k-th nearest are candidates of its tile
    (equivalently: the k-th nearest candidate is nearer than every non-candidate).  Returns the tiles."""
    xy, gx, gy = (np.asarray(a, dtype=np.float64) for a in (xy, gx, gy))
    assert np.all(xy * 16 == np.rint(xy * 16)) and np.all(gx * 16 == np.rint(gx * 16))
    assert np.all(gy * 16 == np.rint(gy * 16))
    k = min(k, len(xy))
    level2 = T.key_level(xy, gx, gy) == 2
    ts = T.tiles(xy, gx, gy, k)
    for row in ts:
        for t in row:
            cand = t.candidates()
            assert cand.sum() >= k
            if cand.all():
                continue
            dc = _grid_d2(xy, gx, gy, t.i0, t.i1, t.j0, t.j1, cand)
            kth = np.partition(dc, k - 1, axis=1)[:, k - 1]
            far = _grid_d2(xy, gx, gy, t.i0, t.i1, t.j0, t.j1, ~cand).min(axis=1)
            bad = np.nonzero(far <= kth)[0]
            assert bad.size == 0, (t.j0, t.i0, t.bk, t.bmax, int(kth[bad[0]]), int(far[bad[0]]))
            if t.key32 and level2:
                # idw32_kernel's key: (4 d^2) << 11 | index, 4 d^2 = dc / 64 from the doubled coordinates
                assert np.all(dc % 64 == 0) and int(np.max(dc)) // 64 < T.KEY32_LIMIT, (t.j0, t.i0)
                assert (int(np.max(dc)) // 64 << 11 | 2047) < 2 ** 32
    return ts


def test_fill_kernel_rule():
    """idw_fill_kernel's table, written out: 20 neighbours take the sorted 64-bit or 32-bit keys while
    the index fits 11 bits, every other k (or fewer vectors than 20) the insertion list."""
    assert T.fill_kernel(20, 0, 2, True) == T.NONE
    for n in (1, 19):
        assert T.fill_kernel(20, n, 2, True) == T.INSERT
    for n in (20, 21, 2047, 2048):
        assert [T.fill_kernel(20, n, lv, f) for lv in (2, 1, 0) for f in (True, False)] == \
            [T.KEY32, T.PACKED, T.PACKED, T.PACKED, T.UNPACKED, T.UNPACKED]
    for n in (2049, 4096, 4097):
        assert {T.fill_kernel(20, n, lv, f) for lv in (2, 1, 0) for f in (True, False)} == {T.UNPACKED}
    for k in list(range(1, 20)) + list(range(21, 33)):
        assert {T.fill_kernel(k, n, lv, True) for n in (1, 21, 2048, 4097) for lv in (0, 1, 2)} == {T.INSERT}
    assert T.fast_weights(2, 0.5, 0.5, 1.0) and not T.fast_weights(2, 0.5, 0.0, 1.0)
    assert not T.fast_weights(3, 0.5, 0.5, 1.0) and not T.fast_weights(2, 1.0, 0.5, 1.0)
    assert not T.fast_weights(2, 0.5, 0.5, 2.0)


def test_cases_reach_their_branches():
    """The claims the GPU edge tests make about their vector sets."""
    for n in T.STRIP_NS:
        xy, gx, gy = T.strip_case(n)
        b = T.tile_bounds(xy, gx, gy, 20)
        declined = np.nonzero(~b["key32"].all(axis=0))[0]
        over = np.nonzero(b["overflow"].any(axis=0))[0]
        assert declined[0] == 49 and over[0] == 89, (n, declined[:3], over[:3])
        assert b["key32"].any() and b["sorted"].all()
        assert T.coverage(xy, gx, gy, 13)[1] > 0
    xy, gx, gy = T.partial_case(17, 17)
    b = T.tile_bounds(xy, gx, gy, 20)
    assert b["overflow"][1, 1] and not b["key32"][1, 1] and b["key32"][0, 0]   # the 1-pixel corner tile
    for ny, nx in T.PARTIAL_GRIDS:
        xy, gx, gy = T.partial_case(ny, nx)
        b = T.tile_bounds(xy, gx, gy, 20)
        if ny % 16 == 1 and nx % 16 == 1:  # a 1-pixel corner tile: r = 0, every vector in the overflow bin
            assert b["overflow"][-1, -1] and not b["key32"][-1, -1], (ny, nx)
    for n in T.CLUSTER_NS:
        xy, gx, gy = T.cluster_case(n)
        assert not T.tile_bounds(xy, gx, gy, 20)["sorted"].any(), n
        assert len(np.unique(xy, axis=0)) < n  # coincident vectors
    assert T.CLUSTER_NS[-1] > T.KD_SHARED_MAX  # the serial tree build of the recomputation
    assert [T.fill_kernel(20, n, 2, True) for n in T.COUNT_NS] == \
        [T.INSERT, T.KEY32, T.KEY32, T.KEY32, T.KEY32, T.UNPACKED, T.UNPACKED, T.UNPACKED]
    forms = []
    for t in T.TRANSLATIONS:
        xy, gx, gy = T.translated_case(t)
        forms.append(T.fill_kernel(20, len(xy), T.key_level(xy, gx, gy), True))
    assert forms == [T.KEY32, T.KEY32, T.KEY32, T.UNPACKED, T.UNPACKED, T.UNPACKED]
    for nx in T.WIDE_NXS:
        xy, gx, gy = T.wide_case(nx)
        assert T.key_level(xy, gx, gy) == 2 and T.coverage(xy, gx, gy, 20)[0] > 0


@pytest.mark.parametrize("name", [c[0] for c in T.gpu_configs() if c[0] != "nonuniform"])
def test_bound_keeps_the_k_nearest_on_the_gpu_cases(name):
    name, xy, gx, gy, ks = next(c for c in T.gpu_configs() if c[0] == name)
    for k in ks:
        _check_bound(xy, gx, gy, k)


def test_bound_on_decreasing_and_degenerate_grids():
    rng = np.random.default_rng(5)
    xy = T.half_points(500, 90, 70, rng, -10.0, -10.0)
    gx, gy = np.arange(81.0), np.arange(61.0)
    for k in (1, 13, 20, 32):
        for a, b in ((gx[::-1], gy), (gx, gy[::-1]), (gx[::-1], gy[::-1]), (gx[:1], gy), (gx, gy[:1]),
                     (gx[:1], gy[:1]), (gx[:17], gy[:1]), (gx[:2], gy[:33])):
            _check_bound(xy, a, b, k)


def test_bound_with_a_tight_triangle_inequality():
    """k coincident vectors beyond one corner of a tile, on the diagonal through its centre, and one
    vector beyond the opposite corner at (or just inside) the k-th distance of that corner pixel: the
    vector's centre distance is the bound's Rk + 2 r exactly."""
    gx, gy = np.arange(16.0), np.arange(16.0)
    for k in (1, 2, 13, 20, 32):
        for far in (0.5, 3.0, 40.0, 700.5):
            for gap in (0.0, 0.5, 1.0):
                xy = np.concatenate([np.full((k, 2), 15.0 + far), [[-(15.0 + far) + gap] * 2]])
                ts = _check_bound(xy, gx, gy, k)
                assert len(ts) == 1 and ts[0][0].candidates()[-1]
                # and the mirror image, with the grid decreasing
                _check_bound(15.0 - xy, gx[::-1], gy[::-1], k)


def test_bound_with_the_kth_distance_on_a_bin_edge():
    """A 1 x 16 tile (the last column of a 17-wide grid: r = 7.5, bin width 3.75) with its vectors at
    multiples of the bin width from the tile centre, on the column through it and off it."""
    gx, gy = np.arange(17.0), np.arange(16.0)
    t = T.tiles(np.zeros((1, 2)), gx, gy, 1)[0][1]
    assert (t.cx, t.cy, t.rt, t.binw) == (16.0, 7.5, 7.5, 3.75)
    for k in (1, 5, 20):
        for m0 in (0, 1, 7, 30):
            ys = 7.5 + 3.75 * np.arange(m0, m0 + k + 3)
            xy = np.concatenate([np.stack([np.full_like(ys, 16.0), ys], 1),
                                 np.stack([16.0 + 3.75 * np.arange(m0, m0 + k + 3), np.full_like(ys, 7.5)], 1),
                                 [[16.0 - 3.75 * (m0 + 6), 7.5]]])
            ts = _check_bound(xy, gx, gy, k)
            assert ts[0][1].bk >= m0


def test_bound_on_random_sixteenth_and_sparse_sets():
    rng = np.random.default_rng(9)
    for n, span, k in ((25, 300, 20), (60, 2000, 20), (21, 40, 20), (700, 120, 32), (3, 50, 1)):
        xy = rng.integers(-16 * span, 16 * span, (n, 2)) / 16.0
        _check_bound(xy, np.arange(-40.0, 57.0), np.arange(10.0, 83.0), k)


def test_packed_keys_leave_the_index_bits_free_at_the_extremes():
    """Level 1 (every coordinate a multiple of 1/16 below 2^14): the squared distance's float64 pattern
    ends in 11 zero bits, also for vectors near -16383.9375 and grid points near +16383.9375."""
    lo = -16383.9375 + np.arange(0, 64) / 16.0
    hi = 16383.9375 - np.arange(0, 64) / 16.0
    for qx in (hi, lo[::-1], np.arange(-40, 40) / 16.0):
        for sx in (lo, hi, np.arange(-40, 40) / 16.0 + 0.0625):
            dx = sx[:, None] - qx[None, :]
            for dy in (dx, dx[::-1], np.zeros_like(dx)):
                d2 = dx * dx + dy * dy
                assert d2.max() < 2.0 ** 31
                assert not np.any(d2.view(np.uint64) & np.uint64(2047))


def test_tie_queries_fit_their_heap():
    """Every tree query the GPU edge tests can issue (all grid points, every k they use) keeps at most
    64 pending nodes (knn.cu QHEAP): none needs the overflow arena."""
    from host_kernels import lib
    L = lib()
    L.host_kd_knn_pairs.restype = ctypes.c_int

    def ptr(a):
        return a.ctypes.data_as(ctypes.c_void_p)

    def overflows(xy, gx, gy, k):
        xy = np.ascontiguousarray(xy, dtype=np.float64)
        GX, GY = np.meshgrid(gx, gy)
        q = np.ascontiguousarray(np.stack([GX.ravel(), GY.ravel()], 1), dtype=np.float64)
        k = min(k, len(xy))
        perm = np.empty(len(xy), dtype=np.int32)
        out = np.empty((len(q), k), dtype=np.int32)
        return L.host_kd_knn_pairs(ptr(xy), len(xy), ptr(q), len(q), k, -1, 64, ptr(perm), ptr(out))

    for name, xy, gx, gy, ks in T.gpu_configs():
        for k in ks:
            assert overflows(xy, gx, gy, k) == 0, (name, k)
    from oracle import lucaskanade as ora
    import warnings
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        sxy, suv = ora.dense_lucaskanade(T.dense_frames(), dense=False)
    dxy, _ = ora.decluster(sxy, suv, 20, 1)
    assert overflows(dxy, np.arange(2048.0), np.arange(256.0), 20) == 0
