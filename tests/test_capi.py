"""CPU tests of the C-ABI boundary: the shared library loads, exports every symbol
declared in include/pysteps_b200.h, the ctypes signature table covers the header,
and the product path refuses to run (loudly) without a GPU instead of falling back."""
import ctypes
import os

import numpy as np
import pytest

from pysteps_b200 import _lib


def test_library_built_and_loads():
    assert os.path.exists(_lib.LIB_PATH), "run `make -C pysteps_b200/csrc` (or __graft_entry__.build())"
    lib = _lib.load()
    assert lib.b200_version() >= 100


def test_every_header_symbol_is_exported_and_bound():
    names = _lib.header_symbols()
    assert len(names) >= 7
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in names:
        assert hasattr(raw, name), f"{name} declared in the header but not exported"
        assert name in _lib._SIGNATURES, f"{name} has no ctypes signature in _lib.py"
    for name in _lib._SIGNATURES:
        assert name in names, f"{name} bound in _lib.py but not declared in the header"


def test_last_error_is_a_string():
    lib = _lib.load()
    msg = lib.b200_last_error()
    assert isinstance(msg, bytes)


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import pysteps_b200
    f = pysteps_b200.extrapolation.get_method("semilagrangian")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        f(np.zeros((8, 8)), np.ones((2, 8, 8)), 1)


def test_product_package_never_imports_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "pysteps_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(d, f)).read()
                assert "import oracle" not in text and "from oracle" not in text, f
                assert "liboracle" not in text, f


def test_get_method_contract():
    # pysteps/tests/test_interfaces.py:58-91 (names, case-insensitivity, errors)
    from pysteps_b200.extrapolation import get_method, semilagrangian, eulerian_persistence
    assert get_method("semilagrangian") is semilagrangian.extrapolate
    assert get_method("SemiLagrangian") is semilagrangian.extrapolate
    assert get_method("eulerian") is eulerian_persistence
    assert get_method(None)(None, None, None) is None
    with pytest.raises(ValueError):
        get_method("nonexistent")
    precip = np.random.rand(10, 10)
    out = eulerian_persistence(precip, None, 3)
    assert out.shape == (3, 10, 10) and np.array_equal(out[2], precip)
    out, disp = eulerian_persistence(precip, None, [1, 2], return_displacement=True)
    assert out.shape == (2, 10, 10) and not disp.any()


def test_sl_entry_points_name_the_first_broken_rule():
    """The semi-Lagrangian entry points check their arguments in a fixed order and report the first
    rule an input breaks, with its error code; unknown dtype codes are named in the message.  Every
    call here is refused before any device work, so no GPU is needed."""
    lib = _lib.load()
    td = np.ones(40)
    tdp = td.ctypes.data_as(_lib.c_dp)
    buf = 0x1000  # a device pointer that is never dereferenced: each call below is refused first
    einval, enotsup = 100001, 100002

    def check(fn, defaults, want_rc, want_msg, **kw):
        args = dict(defaults, **kw)
        rc = getattr(lib, fn)(*args.values())
        msg = lib.b200_last_error().decode().split(" (")[0]
        assert (rc, msg) == (want_rc, want_msg), (fn, kw)

    rows = dict(precip=buf, velocity=buf, xy=None, disp_prev=None, tdiff=tdp, T=4, vts=1.0, n_iter=1, outval=0.0,
                mode=0, vdt=1, layout=0, pdt=1, m=8, n=8, r0=0, rows=8, out=buf, disp_out=None, stream=None)
    f32 = dict(precip=buf, velocity=buf, disp_prev=None, tdiff=tdp, T=4, vts=1.0, outval=0.0, mode=0, vdt=1,
               layout=0, pdt=1, m=8, n=8, r0=0, rows=8, out=buf, disp_out=None, fallback=None, stream=None)
    traj = dict(velocity=buf, xy=None, disp_prev=None, tdiff=tdp, T=4, vts=1.0, n_iter=1, vdt=1, layout=0, m=8,
                n=8, r0=0, rows=8, steps=buf, stream=None)
    for fn, d in (("b200_sl_extrapolate_rows", rows), ("b200_sl_extrapolate_rows_f32", f32),
                  ("b200_sl_trajectories", traj)):
        null = {"b200_sl_extrapolate_rows": "velocity is NULL",
                "b200_sl_extrapolate_rows_f32": "precip, velocity and out are required",
                "b200_sl_trajectories": "velocity / disp_steps is NULL"}[fn]
        check(fn, d, einval, "row band out of range", r0=-1, layout=5, velocity=None)
        check(fn, d, einval, "row band out of range", r0=4, rows=5)
        check(fn, d, einval, "row band out of range", rows=0)
        check(fn, d, einval, "unknown velocity layout", layout=2, velocity=None)
        check(fn, d, einval, null, velocity=None, tdiff=None)
        check(fn, d, einval, "need at least one timestep", tdiff=None, m=8, n=0)
        check(fn, d, einval, "need at least one timestep", T=0)
        check(fn, d, einval, "grid must have 1 .. 2^30 pixels", n=0)
        check(fn, d, einval, "grid must have 1 .. 2^30 pixels", n=1 << 27)
    check("b200_sl_extrapolate_rows_f32", f32, einval, "precip, velocity and out are required", precip=None)
    check("b200_sl_extrapolate_rows_f32", f32, einval, "precip, velocity and out are required", out=None)
    check("b200_sl_trajectories", traj, einval, "velocity / disp_steps is NULL", steps=None)
    for fn, d in (("b200_sl_extrapolate_rows", rows), ("b200_sl_trajectories", traj)):
        check(fn, d, einval, "n_iter must be >= 0", n_iter=-1, **({"mode": 7} if "mode" in d else {}))
    for fn, d in (("b200_sl_extrapolate_rows", rows), ("b200_sl_extrapolate_rows_f32", f32)):
        check(fn, d, einval, "unsupported mode", mode=7, T=33)
        check(fn, d, einval, "unknown field dtypes 7 / 1", vdt=7)
        check(fn, d, einval, "unknown field dtypes 1 / -1", pdt=-1)
    check("b200_sl_extrapolate_rows", rows, einval, "precip and out must both be given or both NULL", out=None)
    check("b200_sl_extrapolate_rows", rows, einval, "precip and out must both be given or both NULL", precip=None)
    check("b200_sl_extrapolate_rows", rows, einval, "nothing to compute", precip=None, out=None)
    check("b200_sl_extrapolate_rows", rows, einval, "unknown field dtypes 2 / 1", precip=None, out=None,
          disp_out=buf, vdt=2)
    check("b200_sl_extrapolate_rows_f32", f32, enotsup, "the float32-tap kernel takes at most 32 timesteps per call",
          T=33, vdt=7)
    check("b200_sl_trajectories", traj, einval, "unknown velocity dtype 4", vdt=4)

    batched = dict(velocity=buf, vdt=1, m=8, n=8, members=3, coefs=buf, vsf=1.0, precip=buf, pdt=1, disp_prev=None,
                   tdiff=1.0, vts=1.0, outval=0.0, mode=0, out=buf, disp_out=buf, nnf=None, stream=None)
    check("b200_sl_step_batched", batched, einval, "unknown field dtypes 0 / 5", vdt=0, pdt=5)
    check("b200_sl_interleave_velocity", dict(velocity=buf, vdt=3, m=8, n=8, out=buf, stream=None), einval,
          "unknown velocity dtype 3")
    bps = dict(velocity=buf, vdt=3, m=8, n=8, a=0.0, b=0.0, vsf=1.0, what=0, out=buf, nnf=None, stream=None)
    check("b200_bps_perturb_velocity", bps, einval, "unknown velocity dtype 3")
