"""GPU parity tests of the device cKDTree (csrc/knn.cu): the warp-parallel build gives scipy's
tree order (oracle/ckdtree.py is pinned against the scipy binary), the outlier stage and the
grid fill follow its neighbour order at exact distance ties.  Branch coverage of the grid fill's tile
search (every search form, far, partial and multi-round tiles, count and key-level boundaries) lives in
test_idw_edges_gpu.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _lib


def _points(kind, n, rng):
    W = int(rng.choice([16, 64, 300, 2048]))
    pts = np.floor(rng.uniform(0, W, (n, 2)))
    if kind == "half":
        pts = np.floor(rng.uniform(0, W, (n, 2)) * 2) / 2
    elif kind == "dup" and n >= 8:
        pts[: n // 4] = pts[n // 4: 2 * (n // 4)]
    elif kind == "few_values":
        pts = np.floor(rng.uniform(0, 4, (n, 2)))
    elif kind == "real":
        pts = rng.uniform(0, W, (n, 2))
    elif kind == "sorted":
        pts = pts[np.lexsort((pts[:, 1], pts[:, 0]))]
    elif kind == "const_x":
        pts[:, 0] = 7.0
    elif kind == "lattice":
        side = int(np.ceil(np.sqrt(n)))
        g = np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2)[:n].astype(np.float64)
        pts = g[rng.permutation(n)] * 10.0
    return np.ascontiguousarray(pts)


@pytest.mark.parametrize("kind", ["int", "half", "dup", "few_values", "real", "sorted", "const_x", "lattice"])
def test_tree_build_matches_scipy_order(env, kind):
    """tree.indices of the device build == the oracle's (== scipy's) for 0 .. 4096 points (shared
    memory build, one warp per node) and above (sequential fallback)."""
    torch, L = env
    from oracle.ckdtree import KDTree
    rng = np.random.default_rng(len(kind))
    s = torch.cuda.current_stream().cuda_stream
    for n in (1, 2, 16, 17, 18, 33, 100, 957, 2000, 4096, 4500):
        pts = _points(kind, n, rng)
        d = torch.from_numpy(pts).cuda()
        idx = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        L.call("b200_kdtree_build", d.data_ptr(), None, n, idx.data_ptr(), cnt.data_ptr(), s)
        torch.cuda.synchronize()
        assert np.array_equal(idx.cpu().numpy(), KDTree(pts).indices), (kind, n)
        # the count on the device (n_dev) path
        nd = torch.tensor([max(n - 3, 1)], dtype=torch.int32, device="cuda")
        L.call("b200_kdtree_build", d.data_ptr(), nd.data_ptr(), n, idx.data_ptr(), cnt.data_ptr(), s)
        torch.cuda.synchronize()
        k = max(n - 3, 1)
        assert np.array_equal(idx.cpu().numpy()[:k], KDTree(pts[:k]).indices), (kind, n, "n_dev")


@pytest.mark.parametrize("kind", ["int", "half", "dup", "few_values", "lattice"])
def test_outlier_flags_follow_ckdtree_order(env, kind):
    torch, L = env
    from oracle import lucaskanade as ora
    rng = np.random.default_rng(7 + len(kind))
    s = torch.cuda.current_stream().cuda_stream
    for n in (2, 3, 10, 40, 300, 1500, 2000):
        xy = _points(kind, n, rng)
        uv = np.stack([2 + 0.3 * rng.standard_normal(n), -1 + 0.3 * rng.standard_normal(n)], 1)
        uv[::7] += 2.0
        for k in (5, 30, 100):
            thr = float(rng.choice([1, 2, 3]))
            duv, dxy = torch.from_numpy(uv).cuda(), torch.from_numpy(xy).cuda()
            flags = torch.empty(n, dtype=torch.uint8, device="cuda")
            L.call("b200_detect_outliers", duv.data_ptr(), dxy.data_ptr(), None, n, thr, k, flags.data_ptr(), s)
            torch.cuda.synchronize()
            with np.errstate(all="ignore"):
                import warnings
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    want = ora.detect_outliers(uv, thr, xy, k)
            assert np.array_equal(flags.cpu().numpy().astype(bool), want), (kind, n, k, thr)


@pytest.mark.parametrize("kind", ["int", "half", "lattice", "real", "dup"])
def test_grid_fill_equals_the_tree_search_everywhere(env, kind):
    """b200_idw_fill (exhaustive tile search + recomputation of the tied grid points) against
    b200_idw_fill_ckdtree (scipy's query at EVERY grid point) and the oracle: <= 1e-12 at every
    grid point, on vector sets where most grid points have an equidistant k-th neighbour."""
    torch, L = env
    from oracle import lucaskanade as ora
    rng = np.random.default_rng(11 + len(kind))
    s = torch.cuda.current_stream().cuda_stream
    for npts, (ny, nx) in ((5, (40, 50)), (21, (64, 64)), (400, (200, 240)), (1500, (300, 310)), (2500, (96, 128))):
        xy = _points(kind, npts, rng)
        xy *= min(1.0, 0.9 * nx / max(xy.max(), 1.0)) if kind == "real" else 1.0
        vals = np.stack([2 + rng.standard_normal(npts), -1 + rng.standard_normal(npts)], 1)
        gx, gy = np.arange(nx, dtype=np.float64), np.arange(ny, dtype=np.float64)
        on_grid = int(kind != "real" and xy.max() < 16384)
        if on_grid and np.all(xy * 2 == np.rint(xy * 2)):
            on_grid = 2  # half-pixel vectors, integer grid: the 32-bit integer-key kernel
        dxy, dv = torch.from_numpy(xy).cuda(), torch.from_numpy(vals).cuda()
        dgx, dgy = torch.from_numpy(gx).cuda(), torch.from_numpy(gy).cuda()
        for k in (20, 8, 13):
            kk = min(k, npts)
            a = torch.empty((2, ny, nx), dtype=torch.float64, device="cuda")
            b = torch.empty((2, ny, nx), dtype=torch.float64, device="cuda")
            L.call("b200_idw_fill", dxy.data_ptr(), dv.data_ptr(), None, npts, 2, kk, 0.5, 0.5, 1.0,
                   dgx.data_ptr(), nx, dgy.data_ptr(), ny, on_grid, a.data_ptr(), s)
            L.call("b200_idw_fill_ckdtree", dxy.data_ptr(), dv.data_ptr(), None, npts, 2, kk, 0.5, 0.5, 1.0,
                   dgx.data_ptr(), nx, dgy.data_ptr(), ny, b.data_ptr(), s)
            torch.cuda.synchronize()
            a, b = a.cpu().numpy(), b.cpu().numpy()
            assert np.abs(a - b).max() <= 1e-12, (kind, npts, k)
            want = ora.idwinterp2d(xy, vals, gx, gy, k=k)
            assert np.abs(b - want).max() <= 1e-13, (kind, npts, k)
            _, tie = ora.idwinterp2d(xy, vals, gx, gy, k=k, return_ties=True)
            if kind in ("int", "lattice") and npts >= 400 and k == 20:
                assert tie.mean() > 0.01  # the case is what it claims to be
        # the general epilogue (another power / offset / resolution): same bar
        a = torch.empty((2, ny, nx), dtype=torch.float64, device="cuda")
        L.call("b200_idw_fill", dxy.data_ptr(), dv.data_ptr(), None, npts, 2, min(20, npts), 1.5, 0.25, 1.0,
               dgx.data_ptr(), nx, dgy.data_ptr(), ny, on_grid, a.data_ptr(), s)
        torch.cuda.synchronize()
        want = ora.idwinterp2d(xy, vals, gx, gy, k=20, power=1.5, dist_offset=0.25)
        assert np.abs(a.cpu().numpy() - want).max() <= 1e-12, (kind, npts)
