"""B200 semi-Lagrangian extrapolation -- drop-in for
``pysteps.extrapolation.semilagrangian.extrapolate``
(pysteps/extrapolation/semilagrangian.py:21-266).

The host side reproduces the reference's argument handling (validation order,
error types and messages, kwargs defaults, return shapes/dtypes); the leadtime
loop -- every ``map_coordinates`` call and NumPy temporary of
semilagrangian.py:181-232 -- is one fused CUDA kernel (``csrc/sl.cu``) reached
through ``b200_sl_extrapolate``.  The input validation reductions
(``np.isfinite`` / ``np.nanmin`` passes, :112-123 and :171-172) run on the
device as well (``b200_field_stats``).

Inputs may be NumPy arrays (results are NumPy arrays, one H2D per input and one
D2H per output) or CUDA ``torch`` tensors (results stay on the device).
"""
import math
import threading
import os
import time
import warnings
import weakref

import numpy as np
import torch

from .. import _device, _lib
from ..noise import motion as _bps

_MODES = {"constant": _lib.MODE_CONSTANT, "nearest": _lib.MODE_NEAREST}

# xy_coords arrays already verified to be the default pixel grid (id -> weakref)
_default_grid_seen = {}


def _is_default_grid(xy_coords, m, n):
    """True when ``xy_coords`` equals the meshgrid of semilagrangian.py:174-179 (what
    nowcasts/steps.py:661-662 and nowcasts/utils.py:361-372 pass), so the kernel can
    generate coordinates from the thread index instead of reading 16 B/pixel."""
    if isinstance(xy_coords, torch.Tensor):
        return False
    key = id(xy_coords)
    ref = _default_grid_seen.get(key)
    xy = np.asarray(xy_coords)
    if ref is not None and ref() is xy_coords:
        # seen before: a few O(1) probes guard against an in-place edit since (corners and centre of
        # both planes); anything else falls through to the full comparison
        if (xy.shape == (2, m, n) and xy[0, 0, 0] == 0 and xy[1, 0, 0] == 0 and xy[0, -1, -1] == n - 1
                and xy[1, -1, -1] == m - 1 and xy[0, m // 2, n // 2] == n // 2 and xy[1, m // 2, n // 2] == m // 2):
            return True
    ok = (xy.shape == (2, m, n)
          and np.array_equal(xy[0], np.broadcast_to(np.arange(n), (m, n)))
          and np.array_equal(xy[1], np.broadcast_to(np.arange(m)[:, None], (m, n))))
    if ok:
        try:
            if len(_default_grid_seen) > 64:
                _default_grid_seen.clear()
            _default_grid_seen[key] = weakref.ref(xy_coords)
        except TypeError:
            pass
    return ok


def _field_tensor(a):
    """Device tensor of a field, keeping float32/float64 storage (anything else -> float64)."""
    if isinstance(a, torch.Tensor):
        dt = a.dtype
    else:
        kept = _device.recall_result(a)  # a field this package returned: still in HBM
        if kept is not None:
            return kept
        a = np.asarray(a)
        dt = a.dtype
    if dt in (np.float32, torch.float32):
        return _device.to_device(a, torch.float32)
    return _device.to_device(a, torch.float64)


_pinned = threading.local()


def _pinned_slot(rows):
    """A small pinned host buffer from a per-thread ring (allocating pinned memory per call costs
    more than the copy it receives)."""
    ring = getattr(_pinned, "ring", None)
    if ring is None:
        ring = _pinned.ring = [torch.empty((4, 4), dtype=torch.float64, pin_memory=True) for _ in range(8)]
        _pinned.next = 0
    if rows > 4:
        return torch.empty((rows, 4), dtype=torch.float64, pin_memory=True)
    _pinned.next = (_pinned.next + 1) % len(ring)
    return ring[_pinned.next][:rows]


def _known_finite(t):
    """A field this package produced and certified finite: its private device copy of a NumPy result
    (`_b200_finite`), or a device tensor handed to the caller that has not been written to since
    (`_b200_finite_version` still equals the tensor's version counter)."""
    if getattr(t, "_b200_finite", False):
        return True
    v = getattr(t, "_b200_finite_version", None)
    return v is not None and v == t._version


def _valid_twin(t, m, n):
    """The (m, n, 2) float64 copy dense_lucaskanade stores beside a device field it returns
    (`_b200_twin`), while the field has not been written to since (`_b200_twin_version` still equals
    its version counter), else None."""
    tw = getattr(t, "_b200_twin", None)
    if tw is None or getattr(t, "_b200_twin_version", None) != t._version:
        return None
    if t.dtype != torch.float64 or tuple(tw.shape) != (m, n, 2):
        return None
    return tw


class _Stats:
    """[(n_nonfinite, nanmin, nanmax, n_nan), ...] of the given fields, reduced on the device.
    The kernels are enqueued at construction.  `post()` -- called once every kernel that writes a
    row has been enqueued, and BEFORE the trajectory kernel is -- enqueues the tiny D2H into pinned
    memory and records an event; `get()` waits for that event only, so the host reads the verdict
    while the trajectory kernel is still running instead of draining the stream."""

    def __init__(self, *tensors):
        self.buf = torch.zeros((len(tensors), 4), dtype=torch.float64, device="cuda")
        s = _device.stream_ptr()
        for i, t in enumerate(tensors):
            # None: the row is filled by the kernel that produces the field.  A remembered result of this
            # package that is finite by construction (the dense LK field) keeps its all-zero row: no scan.
            if t is not None and not _known_finite(t):
                _lib.call("b200_field_stats", t.data_ptr(), _device.dtype_code(t.dtype), t.numel(),
                          self.buf[i].data_ptr(), s)
        self.host = None
        self._pin = self._event = None

    def post(self):
        if self._event is None and self.host is None:
            self._pin = _pinned_slot(self.buf.shape[0])
            self._pin.copy_(self.buf, non_blocking=True)
            self._event = torch.cuda.Event()
            self._event.record()
        return self

    def get(self):
        if self.host is None:
            self.post()
            self._event.synchronize()
            self.host = self._pin.numpy().copy()
        return self.host


def extrapolate(precip, velocity, timesteps, outval=np.nan, xy_coords=None,
                allow_nonfinite_values=False, vel_timestep=1, **kwargs):
    """Semi-Lagrangian backward extrapolation; same contract as the reference
    (see its docstring, semilagrangian.py:30-104).  ``interp_order`` 0..5 as in scipy (order 1 is
    the fused trajectory kernel of csrc/sl.cu, the other orders csrc/spline.cu).  Difference:
    ``map_coordinates_mode`` must be one of "constant"/"nearest" (anything else raises
    NotImplementedError instead of silently using a CPU path).
    """
    if precip is not None and precip.ndim != 2:
        raise ValueError("precip must be a two-dimensional array")

    if velocity.ndim != 3:
        raise ValueError("velocity must be a three-dimensional array")

    _device.require_cuda()
    # `velocity + generate_bps(...)` of pysteps_b200.noise.motion (nowcasts/utils.py:448-451):
    # the perturbed field is produced on the device, directly in the trajectory kernel's layout
    perturbed = isinstance(velocity, _bps.PerturbedVelocity)
    on_device = _device.is_device_tensor(precip) if perturbed else _device.is_device_tensor(velocity)

    d_precip = None if precip is None else _field_tensor(precip)

    # semilagrangian.py:112-123 -- finiteness checks, as device reductions.  Only ENQUEUED here:
    # the verdict is read after the trajectory kernel has been launched (below), so a call costs
    # one host<->device round trip instead of two.  Error precedence is the reference's: a
    # finiteness error outranks every later argument error.
    if perturbed:
        # the producing kernel counts the non-finite elements of the perturbed field itself
        stats = _Stats(*([None] if d_precip is None else [d_precip, None]))
        d_vel = velocity.device_interleaved(stats.buf[-1, 0:1])
        stats.post()
    else:
        d_vel = _field_tensor(velocity)
        stats = _Stats(*([d_vel] if d_precip is None else [d_precip, d_vel])).post()

    def finiteness_errors():
        st = stats.get()
        st_v = st[-1]
        st_p = None if d_precip is None else st[0]
        if not allow_nonfinite_values:
            if st_p is not None and st_p[0] > 0:
                raise ValueError("precip contains non-finite values")
            if st_v[0] > 0:
                raise ValueError("velocity contains non-finite values")
        if st_p is not None and st_p[0] == d_precip.numel():
            raise ValueError("precip contains only non-finite values")
        if st_v[0] == d_vel.numel():
            raise ValueError("velocity contains only non-finite values")

    # warnings of the later stages are held back until the finiteness verdict is in: the
    # reference raises those errors before it warns
    deferred = []
    try:
        result = _extrapolate_checked(precip, velocity, d_precip, d_vel, stats, on_device, timesteps,
                                      outval, xy_coords, vel_timestep, kwargs, deferred,
                                      allow_nonfinite_values)
    except Exception:
        finiteness_errors()  # raises first if the reference would have
        for msg in deferred:
            warnings.warn(msg, stacklevel=2)
        raise
    finiteness_errors()
    for msg in deferred:
        warnings.warn(msg, stacklevel=2)
    return result


# poles of the B-spline prefilters: the doubles nearest to the exact values (decimal literals in
# scipy's ni_splines.c; e.g. sqrt(3.0) - 2.0 evaluated in double is 2 ulp away from the first one)
_POLES = {
    0: (),
    2: (-0.171572875253809902396622551580603843,),                                        # sqrt(8) - 3
    3: (-0.267949192431122706472553658494127633,),                                        # sqrt(3) - 2
    4: (-0.361341225900220177092212841325675255, -0.013725429297339121360331226939128204),
    5: (-0.430575347099973791851434783493520110, -0.043096288203264653822712376822550182),
}
_SPLINE_PAD = 12  # scipy.ndimage._prepad_for_spline_filter, mode "nearest"


def _extrapolate_checked(precip, velocity, d_precip, d_vel, stats, on_device, timesteps, outval,
                         xy_coords, vel_timestep, kwargs, deferred_warnings, allow_nonfinite_values=False):
    """semilagrangian.py:125-266 (everything after the finiteness checks)."""
    if isinstance(timesteps, list) and not sorted(timesteps) == timesteps:
        raise ValueError("timesteps is not in ascending order")

    # defaults (:129-134)
    verbose = kwargs.get("verbose", False)
    displacement_prev = kwargs.get("displacement_prev", None)
    n_iter = kwargs.get("n_iter", 1)
    return_displacement = kwargs.get("return_displacement", False)
    interp_order = kwargs.get("interp_order", 1)
    map_coordinates_mode = kwargs.get("map_coordinates_mode", "constant")
    # extension (ignored by the reference like any unknown kwarg): compute only the output rows
    # [r0, r1) -- results and displacement arrays are then band shaped (tile partitioning of
    # one composite over GPUs; inputs stay full frames)
    rows = kwargs.get("b200_rows", None)
    # extension: sample the fields from float32 copies (values within float32 rounding of the exact
    # path, tap indices certified identical); off by default
    f32_taps = bool(kwargs.get("b200_float32_taps", False))

    if precip is None and not return_displacement:
        raise ValueError("precip is None but return_displacement is False")

    if "D_prev" in kwargs.keys():
        deferred_warnings.append("deprecated argument D_prev is ignored, use displacement_prev instead")

    if interp_order not in (0, 1, 2, 3, 4, 5):
        raise RuntimeError("spline order not supported")  # scipy.ndimage._ni_support._check_order
    if map_coordinates_mode not in _MODES:
        raise NotImplementedError(
            "pysteps_b200 semilagrangian: map_coordinates_mode must be 'constant' or "
            f"'nearest' (got {map_coordinates_mode!r})")

    if isinstance(timesteps, int):
        timesteps = np.arange(1, timesteps + 1)
        vel_timestep = 1.0
    elif np.any(np.diff(timesteps) <= 0.0):
        raise ValueError("the given timestep sequence is not monotonously increasing")

    timestep_diff = np.ascontiguousarray(
        np.hstack([[timesteps[0]], np.diff(timesteps)]), dtype=np.float64)

    if verbose:
        print("Computing the advection with the semi-lagrangian scheme.")
        t0 = time.time()

    # interp_order > 1 (:144-157): the spline runs on a copy whose non-finite values are zeroed
    # (only when they are allowed at all); two order-1 mask warps restore them afterwards
    zero_fill = False
    if precip is not None and interp_order > 1:
        st_p = stats.get()[0]
        if st_p[0] != st_p[3]:
            raise NotImplementedError("pysteps_b200 semilagrangian: interp_order > 1 with +-inf in precip")
        zero_fill = bool(allow_nonfinite_values)

    if precip is not None and isinstance(outval, str) and outval == "min":
        outval = stats.get()[0][1]  # np.nanmin(precip), :171-172
        if zero_fill and stats.get()[0][0] > 0:
            outval = min(outval, 0.0)  # the reference takes it from the zero-filled copy (:150-152)

    m, n = int(velocity.shape[1]), int(velocity.shape[2])
    interleaved = isinstance(velocity, _bps.PerturbedVelocity)
    if velocity.shape[0] != 2:
        raise ValueError("velocity must have shape (2, m, n)")
    if d_precip is not None and tuple(d_precip.shape) != (m, n):
        raise ValueError("precip and velocity have incompatible shapes")

    d_xy = None
    if xy_coords is not None and not _is_default_grid(xy_coords, m, n):
        d_xy = _device.to_device(xy_coords, torch.float64)
        if tuple(d_xy.shape) != (2, m, n):
            raise ValueError("xy_coords must have shape (2, m, n)")

    r0, r1 = (0, m) if rows is None else (int(rows[0]), int(rows[1]))
    if not (0 <= r0 < r1 <= m):
        raise ValueError("b200_rows must satisfy 0 <= r0 < r1 <= m")
    mb = r1 - r0

    d_prev = None
    if displacement_prev is not None:
        d_prev = _device.to_device(displacement_prev, torch.float64)
        if tuple(d_prev.shape) != (2, mb, n):
            raise ValueError("displacement_prev must have shape (2, m, n)")

    T = int(timestep_diff.size)
    d_out = None
    if d_precip is not None:
        d_out = torch.empty((T, mb, n), dtype=d_precip.dtype, device="cuda")
    d_disp = torch.empty((2, mb, n), dtype=torch.float64, device="cuda") \
        if return_displacement else None

    # The library re-lays the field out as (m,n) float64 pairs internally.  While a Trace is
    # active (bench.py / profiling) the re-layout is issued as its own C call so that the
    # trajectory kernel is timed alone.
    layout = _lib.LAYOUT_INTERLEAVED if interleaved else _lib.LAYOUT_PLANAR
    d_v = d_vel
    twin = None if interleaved else _valid_twin(d_vel, m, n)
    if twin is not None:
        # the dense LK field's interleaved copy, written by the fill beside the planar field
        d_v, layout = twin, _lib.LAYOUT_INTERLEAVED
    elif _lib._trace is not None and not interleaved:
        d_v = torch.empty((m, n, 2), dtype=d_vel.dtype, device="cuda")
        _lib.call("b200_sl_interleave_velocity", d_vel.data_ptr(), _device.dtype_code(d_vel.dtype),
                  m, n, d_v.data_ptr(), _device.stream_ptr())
        layout = _lib.LAYOUT_INTERLEAVED
    if f32_taps:
        # opt-in: float32 taps, tap indices certified equal to the exact kernel's (csrc/sl.cu sl_f32_kernel)
        if d_precip is None or interp_order != 1 or n_iter != 1 or d_xy is not None or T > 32:
            raise NotImplementedError(
                "pysteps_b200 semilagrangian: b200_float32_taps needs a precipitation field, interp_order=1, "
                "n_iter=1, the default pixel grid and at most 32 timesteps")
        cnt = kwargs.get("b200_fallback_count", None)  # optional uint64 device tensor, accumulates
        _lib.call("b200_sl_extrapolate_rows_f32",
                  d_precip.data_ptr(), d_v.data_ptr(), _device.ptr(d_prev),
                  timestep_diff.ctypes.data_as(_lib.c_dp), T, float(vel_timestep), float(outval),
                  _MODES[map_coordinates_mode], _device.dtype_code(d_vel.dtype), layout,
                  _device.dtype_code(d_precip.dtype), m, n, r0, mb, d_out.data_ptr(), _device.ptr(d_disp),
                  _device.ptr(cnt), _device.stream_ptr())
    elif d_precip is None or interp_order == 1:
        _lib.call("b200_sl_extrapolate_rows",
                  _device.ptr(d_precip), d_v.data_ptr(), _device.ptr(d_xy), _device.ptr(d_prev),
                  timestep_diff.ctypes.data_as(_lib.c_dp), T, float(vel_timestep),
                  max(int(n_iter), 0),
                  float(outval) if d_precip is not None else 0.0,  # cval is unused without precip (:171-172)
                  _MODES[map_coordinates_mode],
                  _device.dtype_code(d_vel.dtype), layout,
                  _device.dtype_code(d_precip.dtype) if d_precip is not None else _lib.F64,
                  m, n, r0, mb, _device.ptr(d_out), _device.ptr(d_disp), _device.stream_ptr())
    else:
        # spline orders (:224-253): displacement after every leadtime from the trajectory kernel,
        # spline coefficients of the field once (the prefilter sees the same input at every
        # leadtime), then one sampling launch for all leadtimes
        mode = _MODES[map_coordinates_mode]
        pad = _SPLINE_PAD if (interp_order > 1 and map_coordinates_mode == "nearest") else 0
        M, N = m + 2 * pad, n + 2 * pad
        reflect = map_coordinates_mode == "nearest"
        d_steps = torch.empty((T, 2, mb, n), dtype=torch.float64, device="cuda")
        _lib.call("b200_sl_trajectories", d_v.data_ptr(), _device.ptr(d_xy), _device.ptr(d_prev),
                  timestep_diff.ctypes.data_as(_lib.c_dp), T, float(vel_timestep), max(int(n_iter), 0),
                  _device.dtype_code(d_vel.dtype), layout, m, n, r0, mb, d_steps.data_ptr(),
                  _device.stream_ptr())
        d_coeffs = torch.empty((M, N), dtype=torch.float64, device="cuda")
        d_mmin = d_mfin = None
        if interp_order > 1:
            d_mmin = torch.empty((m, n), dtype=torch.float64, device="cuda")
            d_mfin = torch.empty((m, n), dtype=torch.float64, device="cuda")
        d_stats = stats.buf[0]
        poles = np.array(_POLES[int(interp_order)] + (0.0,), dtype=np.float64)
        zp0 = np.array([math.pow(z, M if reflect else M - 1) for z in poles], dtype=np.float64)
        zp1 = np.array([math.pow(z, N if reflect else N - 1) for z in poles], dtype=np.float64)
        _lib.call("b200_spline_prepare", d_precip.data_ptr(), _device.dtype_code(d_precip.dtype), m, n,
                  int(interp_order), mode, d_stats.data_ptr(), int(zero_fill),
                  poles.ctypes.data_as(_lib.c_dp), zp0.ctypes.data_as(_lib.c_dp), zp1.ctypes.data_as(_lib.c_dp),
                  d_coeffs.data_ptr(), _device.ptr(d_mmin), _device.ptr(d_mfin), _device.stream_ptr())
        _lib.call("b200_spline_sample", d_coeffs.data_ptr(), m, n, int(interp_order), mode, _device.ptr(d_xy),
                  d_steps.data_ptr(), T, r0, mb, float(outval), _device.ptr(d_mmin), _device.ptr(d_mfin),
                  d_stats.data_ptr(), _device.dtype_code(d_precip.dtype), d_out.data_ptr(),
                  _device.stream_ptr())
        if d_disp is not None:
            d_disp.copy_(d_steps[T - 1])

    if on_device:
        out, disp = d_out, d_disp
    else:
        out = None if d_out is None else _device.to_host(d_out)
        if d_disp is None:
            disp = None
        elif kwargs.get("b200_resident", False):
            # extension: the displacement is only ever handed back as displacement_prev
            # (nowcasts/utils.py:442-458) -- leave it in HBM, 2 x 32 MB of PCIe per call at 2048^2
            disp = _device.DeviceField(d_disp)
        else:
            disp = _device.to_host(d_disp)

    if verbose:
        torch.cuda.current_stream().synchronize()
        print("--- %s seconds ---" % (time.time() - t0))

    if precip is not None:
        if not return_displacement:
            return out
        return out, disp
    return None, disp


def extrapolate_members(precip, perturbed_velocities, displacement_prev=None, timestep=1.0, vel_timestep=1.0,
                        outval=np.nan, allow_nonfinite_values=False, map_coordinates_mode="constant"):
    """One lead time for ALL ensemble members of this GPU in two launches (extension; the loop body
    of nowcasts/utils.py:440-458 for every member at once).

    Equivalent, member by member and bit for bit, to
        extrapolate(precip[j], perturbed_velocities[j], [timestep], displacement_prev=displacement_prev[j],
                    return_displacement=True, vel_timestep=vel_timestep, ...)
    precip: (M, m, n) stack, NumPy or CUDA tensor (float32 / float64);
    perturbed_velocities: M values of ``velocity + generate_bps(perturbator_j, t)`` from
        ``pysteps_b200.noise`` for perturbators initialised with the SAME velocity array;
    displacement_prev: (M, 2, m, n) from the previous lead time (NumPy, CUDA tensor or the
        DeviceField this function returned) or None at the first.
    Returns (fields (M, m, n), displacement (M, 2, m, n)); CUDA tensors when precip is one.
    """
    _device.require_cuda()
    M = len(perturbed_velocities)
    if M < 1 or not all(isinstance(v, _bps.PerturbedVelocity) for v in perturbed_velocities):
        raise TypeError("perturbed_velocities must be `velocity + generate_bps(...)` handles of pysteps_b200.noise")
    field = perturbed_velocities[0].pert.field
    vsf = perturbed_velocities[0].pert.vsf
    if any(v.pert.field is not field or v.pert.vsf != vsf for v in perturbed_velocities):
        raise ValueError("all members must perturb the same velocity field")
    if map_coordinates_mode not in _MODES:
        raise NotImplementedError("map_coordinates_mode must be 'constant' or 'nearest'")
    if precip.ndim != 3 or precip.shape[0] != M:
        raise ValueError("precip must be an (M, m, n) stack with one field per member")
    _, m, n = (int(v) for v in field.shape)
    if tuple(int(v) for v in precip.shape[1:]) != (m, n):
        raise ValueError("precip and velocity have incompatible shapes")
    on_device = _device.is_device_tensor(precip)
    d_precip = _field_tensor(precip)
    stats = _Stats(d_precip).post()
    coefs = np.ascontiguousarray([[v.pert.a, v.pert.b] for v in perturbed_velocities], dtype=np.float64)
    d_prev = None
    if displacement_prev is not None:
        d_prev = _device.to_device(displacement_prev, torch.float64)
        if tuple(d_prev.shape) != (M, 2, m, n):
            raise ValueError("displacement_prev must have shape (M, 2, m, n)")
    d_out = torch.empty((M, m, n), dtype=d_precip.dtype, device="cuda")
    d_disp = torch.empty((M, 2, m, n), dtype=torch.float64, device="cuda")
    d_bad = torch.empty(M, dtype=torch.float64, device="cuda")
    if isinstance(outval, str) and outval == "min":
        outval = stats.get()[0][1]
    _lib.call("b200_sl_step_batched", field.tensor.data_ptr(), _device.dtype_code(field.tensor.dtype), m, n, M,
              coefs.ctypes.data_as(_lib.c_dp), float(vsf), d_precip.data_ptr(), _device.dtype_code(d_precip.dtype),
              _device.ptr(d_prev), float(timestep), float(vel_timestep), float(outval),
              _MODES[map_coordinates_mode], d_out.data_ptr(), d_disp.data_ptr(), d_bad.data_ptr(),
              _device.stream_ptr())
    st_p = stats.get()[0]
    bad_v = d_bad.cpu().numpy()
    if not allow_nonfinite_values:
        if st_p[0] > 0:
            raise ValueError("precip contains non-finite values")
        if bad_v.any():
            raise ValueError("velocity contains non-finite values")
    if st_p[0] == d_precip.numel():
        raise ValueError("precip contains only non-finite values")
    if on_device:
        return d_out, d_disp
    return _device.to_host(d_out), _device.DeviceField(d_disp)
