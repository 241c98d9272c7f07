"""The kernels each semi-Lagrangian entry point of the C ABI issues: the b200_launch_count() delta of
one direct call on a small grid.  Every re-layout, widening, chunk, batch and fix-up launch is one
count, so a change to the host code that drops, adds or merges a launch shows here."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M, N = 40, 56


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib, _synthetic as syn
    V = syn.velocity_field(M, N, 2, "rotation") * 2.0
    P = syn.rain_field(M, N, 2)
    return dict(torch=torch, lib=_lib, stream=_device.stream_ptr(), V=V, P=P)


def _dev(env, a):
    return env["torch"].from_numpy(np.ascontiguousarray(a)).cuda()


def _launches(env, name, *args):
    lib = env["lib"]
    before = lib.load().b200_launch_count()
    lib.call(name, *args)
    count = lib.load().b200_launch_count() - before
    env["torch"].cuda.synchronize()
    return count


def _velocity(env, dtype, layout):
    V = env["V"].astype(dtype)
    return _dev(env, V if layout == 0 else V.transpose(1, 2, 0))


def _code(dtype):
    return 0 if dtype == np.float32 else 1


@pytest.mark.parametrize("vdtype, layout, pdtype, T, want", [
    (np.float64, 0, np.float64, 40, 3),  # widen + two chunks of at most 32 lead times
    (np.float64, 0, np.float32, 40, 4),  # ... + widen_field
    (np.float64, 1, np.float64, 12, 1),  # the caller's pairs, read as they are
    (np.float32, 1, np.float64, 12, 2),  # widen + one chunk
])
def test_extrapolate_rows(env, vdtype, layout, pdtype, T, want):
    torch = env["torch"]
    vel = _velocity(env, vdtype, layout)
    precip = _dev(env, env["P"].astype(pdtype))
    out = torch.empty((T, M, N), dtype=precip.dtype, device="cuda")
    disp = torch.empty((2, M, N), dtype=torch.float64, device="cuda")
    td = np.ones(T)
    got = _launches(env, "b200_sl_extrapolate_rows", precip.data_ptr(), vel.data_ptr(), None, None,
                    td.ctypes.data_as(env["lib"].c_dp), T, 1.0, 1, float("nan"), 0, _code(vdtype), layout,
                    _code(pdtype), M, N, 0, M, out.data_ptr(), disp.data_ptr(), env["stream"])
    assert got == want


@pytest.mark.parametrize("vdtype, layout, want", [
    (np.float64, 0, 4),  # widen, narrow, float32-tap kernel, fix-up
    (np.float32, 1, 3),  # widen; the caller's float32 pairs are read as they are
    (np.float64, 1, 3),  # narrow; the caller's float64 pairs are read as they are
])
def test_extrapolate_rows_f32(env, vdtype, layout, want):
    torch = env["torch"]
    vel = _velocity(env, vdtype, layout)
    precip = _dev(env, env["P"])
    T = 6
    out = torch.empty((T, M, N), dtype=torch.float64, device="cuda")
    td = np.ones(T)
    got = _launches(env, "b200_sl_extrapolate_rows_f32", precip.data_ptr(), vel.data_ptr(), None,
                    td.ctypes.data_as(env["lib"].c_dp), T, 1.0, float("nan"), 0, _code(vdtype), layout, 1, M, N,
                    0, M, out.data_ptr(), None, None, env["stream"])
    assert got == want


def test_trajectories(env):
    torch = env["torch"]
    vel = _velocity(env, np.float64, 0)
    T = 3
    steps = torch.empty((T, 2, M, N), dtype=torch.float64, device="cuda")
    td = np.ones(T)
    got = _launches(env, "b200_sl_trajectories", vel.data_ptr(), None, None, td.ctypes.data_as(env["lib"].c_dp),
                    T, 1.0, 1, 1, 0, M, N, 0, M, steps.data_ptr(), env["stream"])
    assert got == 4  # widen + one launch per lead time


@pytest.mark.parametrize("pdtype, want", [(np.float64, 4), (np.float32, 6)])
def test_step_batched(env, pdtype, want):
    """11 members: two batches of (perturbation, trajectory) launches, plus widen_field per batch."""
    torch = env["torch"]
    members = 11
    vel = _velocity(env, np.float64, 0)
    precip = _dev(env, np.stack([env["P"]] * members).astype(pdtype))
    coefs = np.linspace(-1.0, 1.0, 2 * members)
    out = torch.empty((members, M, N), dtype=precip.dtype, device="cuda")
    disp = torch.empty((members, 2, M, N), dtype=torch.float64, device="cuda")
    nnf = torch.empty(members, dtype=torch.float64, device="cuda")
    got = _launches(env, "b200_sl_step_batched", vel.data_ptr(), 1, M, N, members, coefs.ctypes.data, 2.0,
                    precip.data_ptr(), _code(pdtype), None, 1.0, 1.0, float("nan"), 0, out.data_ptr(),
                    disp.data_ptr(), nnf.data_ptr(), env["stream"])
    assert got == want


def test_bps_perturb_and_interleave(env):
    torch = env["torch"]
    vel = _velocity(env, np.float64, 0)
    out = torch.empty((M, N, 2), dtype=torch.float64, device="cuda")
    nnf = torch.empty(1, dtype=torch.float64, device="cuda")
    assert _launches(env, "b200_bps_perturb_velocity", vel.data_ptr(), 1, M, N, 0.5, -0.25, 2.0, 0,
                     out.data_ptr(), nnf.data_ptr(), env["stream"]) == 1
    assert _launches(env, "b200_sl_interleave_velocity", vel.data_ptr(), 1, M, N, out.data_ptr(),
                     env["stream"]) == 1
