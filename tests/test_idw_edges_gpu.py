"""The IDW grid fill (csrc/idw.cu, tie recomputation in csrc/knn.cu) at the edges of its tile search:
every search form, tiles the 32-bit keys decline, overflow-bin tiles, partial and 1-pixel tiles, tiles
scanned in several unsorted rounds, the vector counts where the rule changes, every k from 1 to 32,
key-level boundaries and the weighting's edges.  Each case asserts the branch it claims through the
restatement in idw_tiles.py (its host-side checks are tests/test_idw_bound.py) and is held four ways:

  (a) across key levels: b200_idw_fill at every level the coordinates qualify for (2, 1, 0) runs another
      search form over the same (distance, index) lists, summed in the same order: bit-identical fields;
  (b) against the oracle's idwinterp2d (cKDTree order): within BAR of max |values|, same NaN pattern;
  (c) against an exhaustive reference written here (exact integer distances, long-double weights and
      sums) at the grid points whose k-th and (k+1)-th neighbours are not equidistant;
  (d) where the device plan takes the case (at most 4096 vectors, two variables, a pixel grid): the
      planned fill against the read-back path (stages.idwinterp2d), bit for bit, twin included."""
import re

import numpy as np
import pytest

import idw_tiles as T

pytestmark = pytest.mark.gpu

# (b) and (c): |field - reference| <= BAR * max |values|.  Largest seen on an H100 80GB HBM3 (700 W):
# 1.0e-15 against the oracle, 6.9e-16 against the exhaustive reference (general epilogue, all cases).
BAR = 1e-14


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    from pysteps_b200.motion import lucaskanade as lkmod
    _device.require_cuda()
    return torch, _lib, lkmod


def _vals(n, nvar, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return (np.arange(nvar) - 0.5 + rng.standard_normal((n, nvar))) * scale


def _mean_res(gx, gy):
    if len(gx) < 2 or len(gy) < 2:
        return 1.0
    return float(np.mean(np.abs([np.gradient(gx).mean(), np.gradient(gy).mean()])))


def _fill(env, xy, vals, gx, gy, k, power, offset, level, mean_res=None):
    """b200_idw_fill into a NaN-filled (nvar, ny, nx) field"""
    torch, L, _ = env
    n, nvar = vals.shape
    mean_res = _mean_res(gx, gy) if mean_res is None else mean_res
    d = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda() for a in (xy, vals, gx, gy)]
    out = torch.full((nvar, len(gy), len(gx)), float("nan"), dtype=torch.float64, device="cuda")
    L.call("b200_idw_fill", d[0].data_ptr(), d[1].data_ptr(), None, n, nvar, min(k, n), float(power),
           float(offset), mean_res, d[2].data_ptr(), len(gx), d[3].data_ptr(), len(gy), int(level), out.data_ptr(),
           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _levels(xy, gx, gy):
    return [lv for lv in (2, 1, 0) if lv <= T.key_level(xy, gx, gy)]


def _across_levels(env, xy, vals, gx, gy, k, power, offset, what):
    """(a): the field at every qualifying key level; returns it (bit-identical at all of them)"""
    fields = [(lv, _fill(env, xy, vals, gx, gy, k, power, offset, lv)) for lv in _levels(xy, gx, gy)]
    lv0, f0 = fields[0]
    for lv, f in fields[1:]:
        assert f.tobytes() == f0.tobytes(), f"{what}: level {lv} != level {lv0} (k={k}, power={power})"
    return f0


def _oracle(xy, vals, gx, gy, k, power, offset):
    from oracle import lucaskanade as ora
    with np.errstate(all="ignore"):
        want = ora.idwinterp2d(xy, vals, gx, gy, k=k, power=power, dist_offset=offset)
        _, ties = ora.idwinterp2d(xy, vals, gx, gy, k=k, power=power, dist_offset=offset, return_ties=True)
    return want.reshape(vals.shape[1], len(gy), len(gx)), ties


def _exact(xy, vals, gx, gy, k, power, offset, mean_res, flat):
    """The exhaustive reference at grid points `flat` (row-major indices): the k nearest by exact squared
    distance (ties by lower index), weights and sums in long double.  Returns (values (nvar, P), tied)."""
    X = np.rint(xy * 16).astype(np.int64)
    ii, jj = np.divmod(flat, len(gx))
    qx, qy = np.rint(gx[jj] * 16).astype(np.int64), np.rint(gy[ii] * 16).astype(np.int64)
    d2 = (X[None, :, 0] - qx[:, None]) ** 2 + (X[None, :, 1] - qy[:, None]) ** 2  # 1/256 px^2
    n = len(xy)
    k = min(k, n)
    order = np.argsort(d2, axis=1, kind="stable")[:, :k]
    dk = np.take_along_axis(d2, order, axis=1)
    tied = np.zeros(len(flat), dtype=bool)
    if n > k:
        nxt = np.partition(d2, k, axis=1)[:, k]
        tied = nxt == dk[:, -1]
    ld = np.longdouble
    with np.errstate(all="ignore"):
        d = np.sqrt(dk.astype(ld)) / ld(16) / ld(mean_res) + ld(offset)
        w = ld(1) / d ** ld(power)
        ws = w.sum(axis=1)
        out = np.stack([(vals[order, v].astype(ld) * w).sum(axis=1) / ws for v in range(vals.shape[1])])
    return out.astype(np.float64), tied


def _close(got, want, scale, what):
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN pattern"
    ok = ~np.isnan(want)
    err = float(np.abs(got[ok] - want[ok]).max()) / scale if ok.any() else 0.0
    assert err <= BAR, f"{what}: {err:.3e} of max |values|"
    return err


def _check(env, xy, vals, gx, gy, k, power, offset, what, got=None, sample=None):
    """(a), (b) and (c) for one weighting; returns the field"""
    xy, vals = np.asarray(xy, dtype=np.float64), np.asarray(vals, dtype=np.float64)
    gx, gy = np.asarray(gx, dtype=np.float64), np.asarray(gy, dtype=np.float64)
    f = _across_levels(env, xy, vals, gx, gy, k, power, offset, what) if got is None else got
    scale = float(np.abs(vals).max())
    N = len(gx) * len(gy)
    sample = sample or min(6000, max(500, 4_000_000 // len(xy)))  # (c) at every grid point, or a sample
    rng = np.random.default_rng(N)
    flat = np.arange(N) if N <= sample else np.sort(rng.choice(N, sample, replace=False))
    ties = None
    if len(gx) >= 2 and len(gy) >= 2:
        want, ties = _oracle(xy, vals, gx, gy, k, power, offset)
        _close(f, want, scale, what + " vs oracle")
    ref, tied = _exact(xy, vals, gx, gy, k, power, offset, _mean_res(gx, gy), flat)
    if ties is not None:
        assert np.array_equal(tied, ties.ravel()[flat]), what + ": tie masks"
    keep = ~tied
    _close(f.reshape(vals.shape[1], -1)[:, flat[keep]], ref[:, keep], scale, what + " vs exhaustive")
    return f


def _planned(env, xy, uv, m, n, **interp):
    """lucaskanade._fill_planned (as in test_lk_seam_gpu.py) on the declustered vectors xy, uv over the
    m x n pixel grid: (field, twin, plan as read by the host)"""
    torch, _, lkmod = env
    nd = len(xy)
    dxy = torch.from_numpy(np.ascontiguousarray(xy, dtype=np.float64)).cuda()
    duv = torch.from_numpy(np.ascontiguousarray(uv, dtype=np.float64)).cuda()
    dc = torch.tensor([nd, nd, nd, 0], dtype=torch.int32, device="cuda")
    lkmod._pixel_grid(0, n), lkmod._pixel_grid(0, m)
    torch.cuda.synchronize()
    got = lkmod._fill_planned(dict(interp), dc, dxy, duv, nd, m, n, 0, m, False)
    assert got is not None, "the planned path declined the call"
    out, twin, filled = got
    torch.cuda.synchronize()
    assert filled
    return out, twin, lkmod._plan_pin.buf.tolist()


def _planned_vs_read_back(env, xy, uv, m, n, level, what, **interp):
    """(d), plus the plan's key level"""
    torch, _, _ = env
    from pysteps_b200 import stages
    out, twin, plan = _planned(env, xy, uv, m, n, **interp)
    assert plan[4] == 2 and plan[5] == level and plan[6] == len(xy), (what, plan)
    want = stages.idwinterp2d(np.asarray(xy, dtype=np.float64), np.asarray(uv, dtype=np.float64),
                              np.arange(n), np.arange(m), **interp)
    o = out.cpu().numpy()
    assert o.tobytes() == np.ascontiguousarray(want).tobytes(), what + ": planned != read-back"
    assert twin.permute(2, 0, 1).cpu().numpy().tobytes() == o.tobytes(), what + ": twin"
    return o


FAST, GENERAL = (0.5, 0.5), (1.5, 0.25)


def _all_ways(env, xy, gx, gy, k, what, seed, plan=True):
    vals = _vals(len(xy), 2, seed)
    f = _check(env, xy, vals, gx, gy, k, *FAST, what + " fast")
    _check(env, xy, vals, gx, gy, k, *GENERAL, what + " general")
    pixel = np.array_equal(gx, np.arange(len(gx))) and np.array_equal(gy, np.arange(len(gy)))
    if plan and pixel and len(gx) >= 2 and len(gy) >= 2 and len(xy) <= T.KD_SHARED_MAX:
        lv = T.key_level(xy, gx, gy) if max(len(gx), len(gy)) < 16384 else 0
        got = _planned_vs_read_back(env, xy, vals, len(gy), len(gx), lv, what, k=k, power=FAST[0],
                                    dist_offset=FAST[1])
        assert got.tobytes() == f.tobytes(), what + ": planned != b200_idw_fill"
    return vals, f


@pytest.mark.parametrize("n", T.STRIP_NS)
@pytest.mark.parametrize("k", T.STRIP_KS)
def test_strip_far_tiles(env, n, k):
    """48 x 3000: the 32-bit keys decline the tiles beyond ~724 px (the packed kernel fills them over
    tile_done), and the far tiles' k-th vector lies in the overflow bin"""
    xy, gx, gy = T.strip_case(n)
    declined, over, _ = T.coverage(xy, gx, gy, k)
    assert over > 0 and (k != 20 or 0 < declined < 3 * 188)  # some tiles on the 32-bit keys, some not
    assert T.fill_kernel(k, n, 2, True) == (T.KEY32 if k == 20 else T.INSERT)
    _all_ways(env, xy, gx, gy, k, f"strip n={n} k={k}", seed=n + k)


@pytest.mark.parametrize("ny,nx", T.PARTIAL_GRIDS)
def test_partial_and_one_pixel_tiles(env, ny, nx):
    xy, gx, gy = T.partial_case(ny, nx)
    b = T.tile_bounds(xy, gx, gy, 20)
    if ny % 16 == 1 and nx % 16 == 1:
        assert b["overflow"][-1, -1] and not b["key32"][-1, -1]
    for k in (20, 7):
        _all_ways(env, xy, gx, gy, k, f"grid {ny}x{nx} k={k}", seed=ny + nx + k)


@pytest.mark.parametrize("n", T.CLUSTER_NS)
def test_multi_round_tiles_with_coincident_vectors(env, n):
    """every tile holds more than 2048 candidates: unsorted rounds, k-th ties across rounds; above 4096
    vectors the recomputation builds its tree serially"""
    xy, gx, gy = T.cluster_case(n)
    assert T.coverage(xy, gx, gy, 20)[2] == 16
    for k in (20, 13):
        _, f = _all_ways(env, xy, gx, gy, k, f"cluster n={n} k={k}", seed=n + k)
        _, ties = _oracle(xy, _vals(n, 2, 0), gx, gy, k, *FAST)
        assert ties.mean() > 0.05  # the recomputation is exercised


@pytest.mark.parametrize("n", T.COUNT_NS)
def test_vector_counts_at_the_rule_boundaries(env, n):
    xy, gx, gy = T.count_case(n)
    assert len(xy) == n
    _all_ways(env, xy, gx, gy, 20, f"n={n}", seed=n)


def test_every_k_from_1_to_32(env):
    xy, gx, gy = T.mid_case()
    for k in range(1, 33):
        _all_ways(env, xy, gx, gy, k, f"mid k={k}", seed=k)


def test_translation_moves_the_form_not_the_field(env):
    """Distances are exact at every offset: the field at the untied grid points is bit-identical while
    the search form goes from the 32-bit keys (the grid below 2^14) to the unpacked keys."""
    base = {}
    forms = []
    for t in T.TRANSLATIONS:
        xy, gx, gy = T.translated_case(t)
        vals = _vals(len(xy), 2, 3)
        level = T.key_level(xy, gx, gy)
        forms.append(T.fill_kernel(20, len(xy), level, True))
        for power, offset in (FAST, GENERAL):
            f = _fill(env, xy, vals, gx, gy, 20, power, offset, level)
            _check(env, xy, vals, gx, gy, 20, power, offset, f"t={t} power={power}", got=f)
            if t == 0:
                base[power] = f, _oracle(xy, vals, gx, gy, 20, power, offset)[1]
            else:
                f0, ties = base[power]
                assert f.reshape(2, -1)[:, ~ties.ravel()].tobytes() == f0.reshape(2, -1)[:, ~ties.ravel()].tobytes(), t
    assert forms == [T.KEY32] * 3 + [T.UNPACKED] * 3


def test_decreasing_grids_flip_the_field(env):
    xy, gx, gy = T.mid_case()
    vals = _vals(len(xy), 2, 4)
    for k in (20, 13):
        for power, offset in (FAST, GENERAL):
            f = _across_levels(env, xy, vals, gx, gy, k, power, offset, "increasing")
            for flip in ((gx[::-1], gy, (2,)), (gx, gy[::-1], (1,)), (gx[::-1], gy[::-1], (1, 2))):
                g = _across_levels(env, xy, vals, flip[0], flip[1], k, power, offset, f"decreasing {flip[2]}")
                assert g.tobytes() == np.ascontiguousarray(np.flip(f, flip[2])).tobytes(), (k, power, flip[2])


@pytest.mark.parametrize("nx", T.WIDE_NXS)
def test_grid_width_at_the_plans_key_level_limit(env, nx):
    """16 x 16383: the plan keeps level 2; 16 x 16384: grid_ok is false and the plan runs the unpacked keys
    where the read-back path (level 2) runs the 32-bit ones"""
    xy, gx, gy = T.wide_case(nx)
    assert T.coverage(xy, gx, gy, 20)[0] > 0
    vals = _vals(len(xy), 2, nx)
    f = _check(env, xy, vals, gx, gy, 20, *FAST, f"16x{nx}", sample=3000)
    got = _planned_vs_read_back(env, xy, vals, 16, nx, 2 if nx < 16384 else 0, f"16x{nx}", k=20)
    assert got.tobytes() == f.tobytes()


def test_weighting_edges(env):
    """the general epilogue: power 0 .. 3.7, offsets 0 (a vector on a grid point: inf / inf), 0.25, 10,
    values far from unit size, 1, 3 and 8 variables"""
    xy, gx, gy = T.weight_case()
    n = len(xy)
    cases = [(2, 1.0, k, p, 0.5) for p in (0.0, 0.5, 1.0, 2.0, 3.7) for k in (20, 6)]
    cases += [(2, 1.0, k, p, o) for o in (0.0, 0.25, 10.0) for p in (0.5, 1.0) for k in (20, 6)]
    cases += [(2, s, 20, p, o) for s in (1e-3, 1e6) for p, o in (FAST, (2.0, 0.25))]
    cases += [(nv, 1.0, k, p, o) for nv in (1, 3, 8) for p, o in (FAST, GENERAL) for k in (20, 6)]
    for nvar, scale, k, power, offset in cases:
        vals = _vals(n, nvar, nvar + k, scale)
        what = f"nvar={nvar} scale={scale} k={k} power={power} offset={offset}"
        f = _check(env, xy, vals, gx, gy, k, power, offset, what)
        if offset == 0.0:  # NaN where a vector sits on the grid point (the pattern is the oracle's)
            assert np.isnan(f[:, 20, 10]).all(), what


@pytest.mark.parametrize("nchunks", [1, 4, 9, 16])
def test_stages_idwinterp2d_resolution_per_sub_grid(env, nchunks):
    """stages.idwinterp2d on non-uniform grids: the reference interpolates each of the nchunks sub-grids
    (np.array_split of either grid) with that sub-grid's own mean resolution (decorators.py:210-236)."""
    from pysteps_b200 import stages
    xy, gx, gy = T.nonuniform_case()
    vals = _vals(len(xy), 2, nchunks)
    got = stages.idwinterp2d(xy, vals, gx, gy, nchunks=nchunks)
    c = int(nchunks ** 0.5)
    subx = [x for x in np.array_split(gx, c) if x.size] if c > 1 else [gx]
    suby = [y for y in np.array_split(gy, c) if y.size] if c > 1 else [gy]
    want = np.zeros((2, len(gy), len(gx)))
    res = set()
    ix = 0
    for sx in subx:
        iy = 0
        for sy in suby:
            want[:, iy:iy + sy.size, ix:ix + sx.size] = _oracle(xy, vals, sx, sy, 20, 0.5, 0.5)[0]
            res.add(_mean_res(sx, sy))
            iy += sy.size
        ix += sx.size
    assert len(res) == c * c  # every sub-grid has its own resolution
    _close(got, want, float(np.abs(vals).max()), f"nchunks={nchunks}")


def test_dense_lucaskanade_with_rain_at_one_end(env, monkeypatch):
    """256 x 2048 frames with rain only in the columns below 200: the production call reaches the tiles the
    32-bit keys decline and the overflow bin; NumPy call vs the oracle, device call (planned fill) vs the
    NumPy call (read-back fill) bit for bit."""
    import warnings
    torch, _, lkmod = env
    from oracle import lucaskanade as ora
    frames = T.dense_frames()
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        sxy, suv = ora.dense_lucaskanade(frames, dense=False)
        want = ora.dense_lucaskanade(frames)
    dxy, duv = ora.decluster(sxy, suv, 20, 1)
    declined, over, _ = T.coverage(dxy, np.arange(2048.0), np.arange(256.0), 20)
    assert len(dxy) >= 20 and declined > 0 and over > 0
    got = lkmod.dense_lucaskanade(frames.copy())
    _close(got, want, float(np.abs(duv).max()), "dense_lucaskanade vs oracle")
    calls = []
    real_call = lkmod._call
    monkeypatch.setattr(lkmod, "_call", lambda name, *a: (calls.append(name), real_call(name, *a))[1])
    dev = lkmod.dense_lucaskanade(torch.from_numpy(frames).cuda())
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert "b200_idw_fill_planned" in calls and "b200_idw_fill" not in calls
    assert dev.cpu().numpy().tobytes() == got.tobytes()
    assert torch.equal(dev._b200_twin, dev.permute(1, 2, 0))


_NAME = re.compile(r"(idw32_kernel|idw_kernel)<([^>]*)>")


def test_kernel_names_follow_the_rule(env):
    """torch.profiler's kernel names for b200_idw_fill: the templates launched are the ones fill_kernel
    names, so check (a) compares different kernels"""
    from torch.profiler import ProfilerActivity, profile
    expect = {
        T.KEY32: {"idw32_kernel<20>", "idw_kernel<20,true,true,true>"},
        T.PACKED: {"idw_kernel<20,true,true,{f}>"},
        T.UNPACKED: {"idw_kernel<20,true,false,{f}>"},
        T.INSERT: {"idw_kernel<32,false,false,false>"},
    }
    seen = set()
    for n, k, (power, offset), level in ((300, 20, FAST, 2), (300, 20, FAST, 1), (300, 20, FAST, 0),
                                         (300, 20, GENERAL, 2), (300, 20, GENERAL, 0), (2500, 20, FAST, 2),
                                         (300, 13, FAST, 2), (10, 20, FAST, 2)):
        xy, gx, gy = T.count_case(n)
        fastw = T.fast_weights(2, power, offset, 1.0)
        vals = _vals(n, 2, 1)
        _fill(env, xy, vals, gx, gy, k, power, offset, level)  # loaded and warm
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _fill(env, xy, vals, gx, gy, k, power, offset, level)
        names = {"".join(m.group(0).split()) for e in prof.events() for m in [_NAME.search(e.name)] if m}
        form = T.fill_kernel(min(k, n), n, level, fastw)
        want = {s.replace("{f}", "true" if fastw else "false") for s in expect[form]}
        assert names == want, (n, k, level, power, names)
        seen.add((form, fastw))
    assert {f for f, _ in seen} == {T.KEY32, T.PACKED, T.UNPACKED, T.INSERT}
    assert (T.PACKED, False) in seen and (T.UNPACKED, False) in seen
