"""GPU tests of the sparse-vector cleansing of dense LK on the edge grid of tests/sparse_edges.py: each C
entry point (b200_detect_outliers_global, b200_detect_outliers, b200_compact_rows, b200_decluster)
against the oracle, the public stages on their own arguments, and dense_lucaskanade on frame stacks
that reach the serial tree build, the pool above the decluster kernel's capacity and its refusal.

Outlier flags are bit-identical to the oracle (pinned to the reference on the CPU) on every row whose
extended-precision Mahalanobis distance lies outside sparse_edges.MD_MARGIN of the threshold;
compaction and declustering are bit-identical everywhere."""
import warnings

import numpy as np
import pytest

import sparse_edges as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _lib


def _padded(torch, a, cap, fill):
    """a (n, ...) on the device in a (cap, ...) buffer whose rows past n hold `fill`"""
    out = np.full((cap,) + a.shape[1:], fill, dtype=a.dtype)
    out[:len(a)] = a[:cap]
    return torch.from_numpy(out).cuda()


def _count_arg(torch, c):
    return None if c["n_dev"] is None else torch.tensor([c["n_dev"]], dtype=torch.int32, device="cuda")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _oracle_flags(uv, thr, xy=None, k=None):
    from oracle import lucaskanade as ora
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        with ora.knn_mode("ckdtree"):
            return ora.detect_outliers(uv.copy(), thr, None if xy is None else xy.copy(), k)


def _assert_flags(got, want, md, sing, cond, thr, tag):
    tie = E.tie_rows(md, sing, cond, thr)
    assert tie.sum() < max(len(want), 1), tag
    bad = np.nonzero((got != want) & ~tie)[0]
    assert bad.size == 0, (tag, bad[:8], md[bad[:8]])


@pytest.mark.parametrize("tag", list(E.GLOBAL))
def test_global_outlier_entry(env, tag):
    torch, L = env
    c = E.GLOBAL[tag]
    uv, n, cap = E.global_inputs(tag), c["n"], E.n_cap(c)
    duv = _padded(torch, uv, cap, 1e30)  # garbage past the count would swamp the covariance
    flags = torch.full((max(cap, 1),), 7, dtype=torch.uint8, device="cuda")
    s, nd = torch.cuda.current_stream().cuda_stream, _count_arg(torch, c)
    L.call("b200_detect_outliers_global", duv.data_ptr(), _ptr(nd), cap, c["thr"],
           flags.data_ptr(), s)
    got = flags.cpu().numpy()
    assert np.all(got[n:cap] == 7), "rows past the count are written"
    got = got[:n].astype(bool)
    want = _oracle_flags(uv, c["thr"])
    if n < 2:
        assert not got.any()
        return
    _assert_flags(got, want, *E.md_extended(uv), c["thr"], tag)


@pytest.mark.parametrize("tag", list(E.KNN))
def test_knn_outlier_entry(env, tag):
    torch, L = env
    c = E.KNN[tag]
    xy, uv = E.knn_inputs(tag)
    n, cap = c["n"], E.n_cap(c)
    dxy, duv = _padded(torch, xy, cap, -5.0), _padded(torch, uv, cap, 1e30)
    flags = torch.full((max(cap, 1),), 7, dtype=torch.uint8, device="cuda")
    s, nd = torch.cuda.current_stream().cuda_stream, _count_arg(torch, c)
    L.call("b200_detect_outliers", duv.data_ptr(), dxy.data_ptr(), _ptr(nd), cap, c["thr"],
           c["k"], flags.data_ptr(), s)
    got = flags.cpu().numpy()
    assert np.all(got[n:cap] == 7), "rows past the count are written"
    got = got[:n].astype(bool)
    if n < 2:
        assert not got.any()
        return
    want = _oracle_flags(uv, c["thr"], xy, c["k"])
    _assert_flags(got, want, *E.md_extended(uv, E.knn_neighbours(xy, c["k"])), c["thr"], tag)


@pytest.mark.parametrize("tag", list(E.COMPACT))
def test_compact_rows_entry(env, tag):
    torch, L = env
    c = E.COMPACT[tag]
    n, cap = c["n"], E.n_cap(c)
    rng = np.random.default_rng(n + 3)
    xy, uv = rng.standard_normal((cap, 2)), rng.standard_normal((cap, 2))
    drop = np.zeros(cap, np.uint8)
    drop[:n] = E.compact_drop(c, np.random.default_rng(0))
    oxy = torch.full((max(cap, 1), 2), np.nan, dtype=torch.float64, device="cuda")
    ouv = torch.full((max(cap, 1), 2), np.nan, dtype=torch.float64, device="cuda")
    cnt = torch.full((1,), -9, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    dxy, duv, ddrop, nd = (torch.from_numpy(xy).cuda(), torch.from_numpy(uv).cuda(), torch.from_numpy(drop).cuda(),
                           _count_arg(torch, c))
    L.call("b200_compact_rows", dxy.data_ptr(), duv.data_ptr(), ddrop.data_ptr(), _ptr(nd), cap, oxy.data_ptr(),
           ouv.data_ptr(), cnt.data_ptr(), s)
    keep = drop[:n] == 0
    k = int(cnt.item())
    assert k == keep.sum()
    assert np.array_equal(oxy.cpu().numpy()[:k], xy[:n][keep]) and np.array_equal(ouv.cpu().numpy()[:k], uv[:n][keep])
    assert np.isnan(oxy.cpu().numpy()[k:]).all(), "rows past the count are written"


def _decluster_call(torch, L, xy, uv, scale, min_samples, n_dev=None, cap=None):
    cap = len(xy) if cap is None else cap
    dxy, duv = _padded(torch, xy, cap, 3.0), _padded(torch, uv, cap, 1e30)
    oxy = torch.full((cap, 2), -7.0, dtype=torch.float64, device="cuda")
    ouv = torch.full((cap, 2), -7.0, dtype=torch.float64, device="cuda")
    cnt = torch.full((1,), -9, dtype=torch.int32, device="cuda")
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    L.call("b200_decluster", dxy.data_ptr(), duv.data_ptr(), _ptr(nd), cap, float(scale), int(min_samples),
           oxy.data_ptr(), ouv.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream().cuda_stream)
    k = int(cnt.item())
    return k, oxy.cpu().numpy(), ouv.cpu().numpy()


@pytest.mark.parametrize("tag", list(E.DECLUSTER))
def test_decluster_entry(env, tag):
    """Bit-identical to the reference's per-cell medians in np.unique(axis=0) order (the vectorised
    restatement, pinned to the reference on the CPU), or refused with a count of -1 and nothing else
    written; with the count on the device as well where the capacity allows garbage rows past it."""
    torch, L = env
    c = E.DECLUSTER[tag]
    xy, uv = E.decluster_inputs(c)
    refused = E.decluster_refused(xy, c["scale"], c["min_samples"])
    want = None if refused else E.decluster_vectorised(xy, uv, c["scale"], c["min_samples"])
    calls = [dict()]
    if c["n"] + E.PAD <= E.DC_MAX:
        calls.append(dict(n_dev=c["n"], cap=c["n"] + E.PAD))
    for kw in calls:
        k, oxy, ouv = _decluster_call(torch, L, xy, uv, c["scale"], c["min_samples"], **kw)
        if refused:
            assert k == -1 and (oxy == -7.0).all() and (ouv == -7.0).all(), (tag, kw)
            continue
        assert k == len(want[0]), (tag, kw, k, len(want[0]))
        assert np.array_equal(oxy[:k], want[0]) and np.array_equal(ouv[:k], want[1]), (tag, kw)
        assert (oxy[k:] == -7.0).all(), (tag, kw)


def test_decluster_capacity(env):
    """DC_MAX vectors are declustered; DC_MAX + 1 are refused by the host before any launch."""
    torch, L = env
    rng = np.random.default_rng(4)
    xy = rng.integers(0, 3000, (E.DC_OVER, 2)).astype(np.float64)
    uv = rng.standard_normal((E.DC_OVER, 2))
    with pytest.raises(RuntimeError, match="at most 16384 vectors"):
        _decluster_call(torch, L, xy, uv, 20.0, 1)
    k, oxy, ouv = _decluster_call(torch, L, xy[:E.DC_MAX], uv[:E.DC_MAX], 20.0, 1)
    want = E.decluster_vectorised(xy[:E.DC_MAX], uv[:E.DC_MAX], 20.0, 1)
    assert k == len(want[0]) and np.array_equal(oxy[:k], want[0]) and np.array_equal(ouv[:k], want[1])


def test_decluster_findings(env):
    """The two cells of x = 3e6 and x = 902848 (scale 1) stay two cells; a NaN row is dropped and +inf
    rows form the last cell, as in the reference."""
    torch, L = env
    k, oxy, ouv = _decluster_call(torch, L, np.array([[3e6, 0.0], [902848.0, 0.0]]), np.arange(4.0).reshape(2, 2),
                                  1.0, 1)
    assert k == 2 and np.array_equal(oxy[:2], [[902848.0, 0.0], [3e6, 0.0]]) and np.array_equal(ouv[:2], [[2, 3], [0, 1]])
    coord = np.array([[1, 1], [np.nan, 2], [1, 2], [np.inf, 3], [np.inf, 5]], float)
    k, oxy, ouv = _decluster_call(torch, L, coord, np.arange(10.0).reshape(5, 2), 20.0, 1)
    assert k == 2 and np.array_equal(oxy[:2], [[1, 1.5], [np.inf, 4]]) and np.array_equal(ouv[:2], [[2, 3], [7, 8]])


@pytest.mark.parametrize("tag", ["g-n2", "g-n257", "g-swap", "g-collinear", "k-lattice1500-k30",
                                 "k-half4097-k30", "k-constx2000-k100", "k-n2", "k-identical-uv"])
def test_public_detect_outliers(env, tag):
    from pysteps_b200 import stages
    c = E.ALL_CASES[tag]
    if c["op"] == "global":
        uv, xy, k = E.global_inputs(tag), None, None
        md = E.md_extended(uv)
    else:
        (xy, uv), k = E.knn_inputs(tag), c["k"]
        md = E.md_extended(uv, E.knn_neighbours(xy, k))
    got = stages.detect_outliers(uv, c["thr"], xy, k)
    assert got.dtype == bool and got.shape == (len(uv),)
    _assert_flags(got, _oracle_flags(uv, c["thr"], xy, k), *md, c["thr"], tag)


@pytest.mark.parametrize("tag", ["d-n1", "d-n2-even", "d-n4096-ms2", "d-negative", "d-roundedge", "d-ms0",
                                 "d-ms-gt-n", "d-beyond2^20", "d-near2^24", "d-beyond2^24", "d-nonfinite",
                                 "d-nan-ms0"])
def test_public_decluster(env, tag):
    from pysteps_b200 import stages
    c = E.DECLUSTER[tag]
    xy, uv = E.decluster_inputs(c)
    if E.decluster_refused(xy, c["scale"], c["min_samples"]):
        with pytest.raises(ValueError, match="decluster"):
            stages.decluster(xy, uv, c["scale"], c["min_samples"])
        return
    got = stages.decluster(xy, uv, c["scale"], c["min_samples"])
    want = E.decluster_vectorised(xy, uv, c["scale"], c["min_samples"])
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


# ----------------------------------------------------------------------------- dense_lucaskanade
def _stack(m, n, T, seed):
    from pysteps_b200 import _synthetic as syn
    return syn.rain_frames(m, n, T, seed, dx=2, dy=-1)


@pytest.mark.parametrize("kw", [dict(), dict(k_outlier=None), dict(k_outlier=31), dict(k_outlier=32),
                                dict(decl_scale=1), dict(decl_scale=0.5), dict(decl_scale=7.5)])
def test_dense_lucaskanade_pool_above_the_shared_tree(env, kw):
    """Six frames, 1000 corners each: a pool of 5000 vectors takes the serial tree build and the
    read-back fill; the sparse vectors are bit-identical and the field within 1e-12 of the oracle."""
    from oracle import lucaskanade as ora
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    fr = _stack(160, 200, 6, 21)
    sxy, suv = lk(fr, dense=False, **kw)
    with ora.knn_mode("ckdtree"):
        oxy, ouv = ora.dense_lucaskanade(fr, dense=False, **kw)
        Vo = ora.dense_lucaskanade(fr, **kw)
    assert np.array_equal(sxy, oxy) and np.array_equal(suv, ouv), kw
    V = lk(fr, **kw)
    assert V.shape == Vo.shape and np.abs(V - Vo).max() <= 1e-12, kw


def test_dense_lucaskanade_pool_above_the_decluster_capacity(env):
    """max_corners 5000 over five frames: a pool of 20000 > DC_MAX with far fewer survivors takes the
    extra count read-back and declusters them."""
    from oracle import lucaskanade as ora
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    fr = _stack(128, 160, 5, 22)
    kw = dict(fd_kwargs=dict(max_corners=5000), decl_scale=6.5)
    V = lk(fr, **kw)
    with ora.knn_mode("ckdtree"):
        Vo = ora.dense_lucaskanade(fr, **kw)
    assert V.shape == Vo.shape and np.abs(V - Vo).max() <= 1e-12


def test_dense_lucaskanade_refuses_more_survivors_than_the_decluster_kernel_holds(env):
    """More than DC_MAX vectors survive the outlier test: NotImplementedError naming the count."""
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    f = syn.powerlaw_field(512, 512, 3)
    f = np.where(f > -1.0, f + 2.0, 0.0)
    fr = np.stack([np.roll(f, (t, 2 * t), (0, 1)) for t in range(4)])
    with pytest.raises(NotImplementedError, match="declustering more than 16384"):
        lk(fr, fd_kwargs=dict(max_corners=30000, min_distance=1, quality_level=1e-3), k_outlier=None,
           nr_std_outlier=50.0)
