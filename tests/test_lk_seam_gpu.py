"""The seam between dense_lucaskanade's sparse stages and the extrapolator: the device plan of the
interpolation stage (b200_idw_plan + b200_idw_fill_planned: no read-back before the fill) and the
interleaved twin of the field that the extrapolator reads instead of re-laying the field out.

Every case is held against the read-back path: pysteps_b200.stages.idwinterp2d (host checks, then
b200_idw_fill / b200_fill_f64 -- the path dense_lucaskanade takes for NumPy results) bit for bit,
errors included, and against the oracle's idwinterp2d."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200.motion import lucaskanade as lkmod
    return torch, lkmod


def _log_syncs(monkeypatch, torch, lkmod):
    """Record the C calls of dense_lucaskanade and every host wait, in order."""
    log = []
    real_call = lkmod._call
    monkeypatch.setattr(lkmod, "_call", lambda name, *a: (log.append(name), real_call(name, *a))[1])
    for cls in (torch.cuda.Event, torch.cuda.Stream):
        real = cls.synchronize
        monkeypatch.setattr(cls, "synchronize", lambda self, _r=real: (log.append("sync"), _r(self))[1])
    return log


def _planned(env, monkeypatch, xy, uv, m, n, counts=None, cap=None, **interp):
    """lucaskanade._fill_planned on the given declustered vectors; vectors beyond the count are NaN and
    must be ignored.  Returns (result or (exception type, message), the plan as read by the host)."""
    torch, lkmod = env
    nd = len(xy)
    cap = max(cap or nd, 1)
    dxy = torch.full((cap, 2), float("nan"), dtype=torch.float64, device="cuda")
    duv = torch.full((cap, 2), float("nan"), dtype=torch.float64, device="cuda")
    if nd:
        dxy[:nd] = torch.from_numpy(np.asarray(xy, dtype=np.float64))
        duv[:nd] = torch.from_numpy(np.asarray(uv, dtype=np.float64))
    c = (max(nd, 1), nd, nd) if counts is None else counts
    dc = torch.tensor(list(c) + [0], dtype=torch.int32, device="cuda")
    lkmod._pixel_grid(0, n), lkmod._pixel_grid(0, m)  # built once per shape (that build waits)
    torch.cuda.synchronize()
    log = _log_syncs(monkeypatch, torch, lkmod)
    try:
        got = lkmod._fill_planned(dict(interp), dc, dxy, duv, cap, m, n, 0, m, False)
    except ValueError as e:
        got = (type(e).__name__, str(e))
    monkeypatch.undo()
    assert got is not None, "the planned path declined the call"
    # nothing is read back before the fill is enqueued
    assert "b200_idw_fill_planned" in log and "sync" in log
    assert log.index("b200_idw_fill_planned") < log.index("sync"), log
    return got, lkmod._plan_pin.buf.tolist()


def _readback(xy, uv, m, n, **interp):
    from pysteps_b200 import stages
    try:
        return stages.idwinterp2d(np.asarray(xy, dtype=np.float64), np.asarray(uv, dtype=np.float64),
                                  np.arange(n), np.arange(m), **interp)
    except ValueError as e:
        return type(e).__name__, str(e)


def _check_field(env, got, want, what):
    torch, _ = env
    out, twin, filled = got
    assert filled, what
    o = out.cpu().numpy()
    assert o.shape == want.shape and np.array_equal(o, want), what
    assert o.tobytes() == np.ascontiguousarray(want).tobytes(), what + " (signed zeros)"
    assert torch.equal(twin, out.permute(1, 2, 0)), what + ": twin != field"
    assert twin.permute(2, 0, 1).cpu().numpy().tobytes() == o.tobytes(), what + ": twin bits"


def test_early_outs_zero_fields(env, monkeypatch):
    torch, _ = env
    xy, uv = np.array([[3.0, 4.0], [10.5, 2.0]]), np.array([[1.0, 2.0], [3.0, -1.0]])
    for counts in ((0, 0, 0), (5, 3, 0), (0, 0, 2)):
        (out, twin, filled), plan = _planned(env, monkeypatch, xy if counts[2] else [], uv if counts[2] else [],
                                             37, 41, counts=counts, cap=4)
        assert not filled and plan[4] == 0 and plan[6] == 0, (counts, plan)
        assert not out.any() and not twin.any() and out.shape == (2, 37, 41) and twin.shape == (37, 41, 2)


@pytest.mark.parametrize("uv0", [(1.5, -2.25), (0.0, -0.0), (-0.0, 0.0)])
def test_one_vector_is_a_constant_field(env, monkeypatch, uv0):
    got, plan = _planned(env, monkeypatch, [[7.0, 9.5]], [uv0], 30, 33, cap=6)
    assert plan[4] == 1, plan
    _check_field(env, (got[0], got[1], True), _readback([[7.0, 9.5]], [uv0], 30, 33), f"one vector {uv0}")


def test_uniform_values_are_a_constant_field(env, monkeypatch):
    rng = np.random.default_rng(1)
    xy = rng.integers(0, 60, (40, 2)) / 2.0
    for val in (1.25, -0.0, 0.0):
        uv = np.full((40, 2), val)
        uv[3, 1] = 0.0 if val == -0.0 else uv[3, 1]  # -0.0 == 0.0: still uniform, first value written
        got, plan = _planned(env, monkeypatch, xy, uv, 50, 64, cap=100)
        assert plan[4] == 1, plan
        _check_field(env, (got[0], got[1], True), _readback(xy, uv, 50, 64), f"uniform {val}")


def test_non_finite_inputs_raise_the_read_back_paths_errors(env, monkeypatch):
    rng = np.random.default_rng(2)
    xy = rng.integers(0, 60, (30, 2)) / 2.0
    uv = rng.standard_normal((30, 2))
    cases = []
    for bad_uv, bad_xy in ((np.nan, None), (np.inf, None), (None, np.nan), (None, -np.inf), (np.nan, np.inf)):
        x, u = xy.copy(), uv.copy()
        if bad_uv is not None:
            u[17, 1] = bad_uv
        if bad_xy is not None:
            x[4, 0] = bad_xy
        cases.append((x, u))
    x1, u1 = xy[:1].copy(), uv[:1].copy()
    u1[0, 0] = np.nan
    cases.append((x1, u1))  # one vector, non-finite: the check comes before the constant fill
    for x, u in cases:
        got, plan = _planned(env, monkeypatch, x, u, 40, 40, cap=64)
        want = _readback(x, u, 40, 40)
        assert isinstance(want, tuple) and got == want, (got, want)
        assert plan[4] == 3, plan


@pytest.mark.parametrize("kind,npts,k,power,offset,level", [
    ("half", 300, 20, 0.5, 0.5, 2),      # 32-bit keys (the usual dense_lucaskanade case)
    ("half", 20, 20, 0.5, 0.5, 2),
    ("sixteenth", 300, 20, 0.5, 0.5, 1),  # packed 64-bit keys
    ("general", 300, 20, 0.5, 0.5, 0),    # unpacked 64-bit keys
    ("half", 2500, 20, 0.5, 0.5, 2),      # more vectors than the packed index holds: unpacked
    ("half", 7, 20, 0.5, 0.5, 2),         # fewer vectors than k: insertion list
    ("half", 100, 8, 0.5, 0.5, 2),        # k = 8: the insertion list on both paths
    ("general", 20, 25, 0.5, 0.5, 0),     # k > npts == 20: the K = 20 kernels
    ("half", 100, 25, 0.5, 0.5, 2),       # k = 25
    ("half", 300, 20, 1.5, 0.25, 2),      # general weights
    ("general", 300, 1, 2.0, 0.5, 0),
])
def test_interpolation_paths_match_the_read_back_path(env, monkeypatch, kind, npts, k, power, offset, level):
    from oracle import lucaskanade as ora
    rng = np.random.default_rng(npts + 7 * k)
    m, n = 120, 131
    if kind == "half":
        xy = rng.integers(-20, 2 * 140, (npts, 2)) / 2.0
    elif kind == "sixteenth":
        xy = rng.integers(-80, 16 * 130, (npts, 2)) / 16.0
    else:
        xy = rng.uniform(-5, 135, (npts, 2))
    uv = rng.standard_normal((npts, 2))
    interp = dict(k=k, power=power, dist_offset=offset)
    got, plan = _planned(env, monkeypatch, xy, uv, m, n, cap=max(npts, 1000), **interp)
    assert plan[4] == 2 and plan[5] == level and plan[6] == npts, plan
    want = _readback(xy, uv, m, n, **interp)
    _check_field(env, got, want, f"{kind} npts={npts} k={k}")
    if npts <= 300:
        assert np.abs(want - ora.idwinterp2d(xy, uv, np.arange(n), np.arange(m), **interp)).max() <= 1e-11


def _case_frames():
    from lk_cases import build_case
    from pysteps_b200 import _synthetic as syn
    out = [(name,) + tuple(build_case(name)) for name in ("plain_160x200", "nan_200x176", "three_frames_192x160",
                                                          "odd_width_150x203")]
    fr = syn.rain_frames(128, 160, 2, 6)
    out += [("one_vector", fr, dict(fd_kwargs=dict(max_corners=1))),
            ("all_outliers", fr, dict(nr_std_outlier=0)),
            ("no_rain", np.zeros((2, 80, 90)), {}),
            ("k8_power", fr, dict(interp_kwargs=dict(k=8, power=1.5))),
            ("band", fr, dict(interp_kwargs=dict(b200_rows=(20, 77))))]
    return out


def test_dense_lucaskanade_device_equals_numpy_path(env, monkeypatch):
    """Device-resident calls (planned fill) against NumPy calls (read-back path) of the same frames:
    identical fields, and the fill enqueued before the host waits for anything."""
    torch, lkmod = env
    for name, frames, kw in _case_frames():
        want = lkmod.dense_lucaskanade(frames.copy(), **kw)
        dfr = torch.from_numpy(np.ascontiguousarray(frames, dtype=np.float64)).cuda()
        lkmod.dense_lucaskanade(dfr, **kw)
        torch.cuda.synchronize()
        log = _log_syncs(monkeypatch, torch, lkmod)
        got = lkmod.dense_lucaskanade(dfr, **kw)
        monkeypatch.undo()
        assert isinstance(got, torch.Tensor) and got.is_cuda, name
        g = got.cpu().numpy()
        assert g.shape == want.shape and g.tobytes() == want.tobytes(), name
        assert "b200_idw_fill_planned" in log, name
        after = log[log.index("b200_decluster"):] if "b200_decluster" in log else log
        assert after.index("b200_idw_fill_planned") < after.index("sync"), (name, log)
        assert torch.equal(got._b200_twin, got.permute(1, 2, 0)), name
    # sparse results and k=None keep the read-back path
    dfr = torch.from_numpy(_case_frames()[0][1]).cuda()
    log = _log_syncs(monkeypatch, torch, lkmod)
    lkmod.dense_lucaskanade(dfr, dense=False)
    lkmod.dense_lucaskanade(dfr, interp_kwargs=dict(k=None))
    monkeypatch.undo()
    assert "b200_idw_fill_planned" not in log


def test_twin_is_used_while_valid_and_ignored_after_a_write(env):
    torch, lkmod = env
    import pysteps_b200
    from pysteps_b200 import _lib
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200.extrapolation import semilagrangian as slmod
    extrap = pysteps_b200.extrapolation.get_method("semilagrangian")
    frames = syn.rain_frames(192, 224, 2, 1)
    P = torch.from_numpy(frames[-1]).cuda()
    V = lkmod.dense_lucaskanade(torch.from_numpy(frames).cuda())
    assert slmod._valid_twin(V, 192, 224) is V._b200_twin
    with _lib.Trace() as tr:
        with_twin, d1 = extrap(P, V, 3, return_displacement=True)
    assert "b200_sl_interleave_velocity" not in tr.summary()
    with _lib.Trace() as tr:
        without, d2 = extrap(P, V.clone(), 3, return_displacement=True)
    assert "b200_sl_interleave_velocity" in tr.summary()
    no_trace, d3 = extrap(P, V.clone(), 3, return_displacement=True)
    for a in (without, no_trace):
        assert torch.equal(torch.nan_to_num(with_twin, nan=-1.0), torch.nan_to_num(a, nan=-1.0))
    assert torch.equal(d1, d2) and torch.equal(d1, d3)
    # an in-place write retires the twin (and the finiteness certificate): the written value is advected
    V[0] += 0.5
    assert slmod._valid_twin(V, 192, 224) is None
    got = extrap(P, V, 3)
    want = extrap(P, V.clone(), 3)
    assert torch.equal(torch.nan_to_num(got, nan=-1.0), torch.nan_to_num(want, nan=-1.0))
    assert not torch.equal(torch.nan_to_num(got, nan=-1.0), torch.nan_to_num(with_twin, nan=-1.0))
    V[1, 5, 7] = float("nan")
    with pytest.raises(ValueError, match="velocity contains non-finite"):
        extrap(P, V, 2)
