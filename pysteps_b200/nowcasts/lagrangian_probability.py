"""B200 local Lagrangian probability nowcast -- drop-in for
``pysteps.nowcasts.lagrangian_probability.forecast`` (pysteps/nowcasts/lagrangian_probability.py).

The probability of exceeding a threshold in a disk neighbourhood of every extrapolated field, the
disk's diameter growing with lead time.  The extrapolation is the device extrapolator
(``extrapolation/semilagrangian.py``), called with device tensors so that its field never leaves
HBM; the neighbourhood step is ``b200_probability`` (csrc/probability.cu).  The argument flow,
exceptions and their order are the reference's (lagrangian_probability.py:69-107 and
nowcasts/extrapolation.py:69-117).

One deviation: the reference's two ``scipy.signal.convolve`` calls per lead run as float32 FFTs
and are off the exact counts by up to a few 1e-7; the device counts are exact integers, so its
probabilities are the exact ratios (within 1e-6 of the reference's).

NumPy input returns a NumPy (T, m, n) float64 array; a CUDA-tensor precip returns a CUDA float64
tensor.

Parity: tests/test_probability_gpu.py (device), tests/test_oracle_probability.py and
tests/test_host_logic_probability.py (oracle and host logic on the CPU).
"""
import numpy as np
import torch

from .. import _compare, _device, _lib
from ..extrapolation import interface as _extrapolation
from ..extrapolation import semilagrangian as _sl
from . import extrapolation as _extrapolation_nowcast

_MAX_SCALE = 1 << 24  # B200_PROBABILITY_MAX_SCALE


def forecast(precip, velocity, timesteps, threshold, extrap_method="semilagrangian", extrap_kwargs=None,
             slope=5):
    """Same contract as the reference: precip (m, n), velocity (2, m, n), timesteps an int > 0 or a
    sorted list, threshold a float; returns P(precip >= threshold) of shape (len(timesteps), m, n).
    Only float32 and float64 fields are supported."""
    if isinstance(timesteps, int) and timesteps > 0:
        timesteps = np.arange(1, timesteps + 1)
    elif not isinstance(timesteps, list):
        raise ValueError(f"invalid value for argument 'timesteps': {timesteps}")

    _extrapolation_nowcast.check_inputs(precip, velocity, timesteps)

    lib = torch if isinstance(precip, torch.Tensor) else np
    if precip.dtype not in (lib.float32, lib.float64):
        raise NotImplementedError(f"pysteps_b200 lagrangian_probability: fields of dtype {precip.dtype} are not "
                                  "supported (float32 or float64)")
    m, n = (int(k) for k in precip.shape)
    if m * n >= 1 << 31:
        raise NotImplementedError("pysteps_b200 lagrangian_probability: frames of 2^31 pixels or more are not "
                                  "supported")

    extrap_kwargs = dict() if extrap_kwargs is None else extrap_kwargs.copy()
    _device.require_cuda()
    on_device = _device.is_device_tensor(precip)
    d_precip = _sl._field_tensor(precip)
    # np.any(~np.isfinite(precip)) as a device reduction
    extrap_kwargs["allow_nonfinite_values"] = bool(_sl._Stats(d_precip).get()[0][0] > 0)

    method = _extrapolation.get_method(extrap_method)
    if method is _sl.extrapolate:
        F = method(d_precip, _extrapolation_nowcast.device_velocity(velocity), timesteps, **extrap_kwargs)
    elif method is _extrapolation.eulerian_persistence and not extrap_kwargs.get("return_displacement", False):
        F = d_precip.unsqueeze(0).expand(len(timesteps), m, n)  # plane stride 0: the field is not replicated
    else:
        F = method(precip, velocity, timesteps, **extrap_kwargs)
    if not isinstance(F, torch.Tensor):
        _fail_as_the_reference(F, threshold)

    plane_stride = F.stride(0)
    T, mf, nf = (int(k) for k in F.shape)  # b200_rows (an extrapolator extension) gives a band
    threshold_cmp, nan_exceeds = _threshold_rule(F.dtype, threshold)
    scales = _scales(timesteps, slope, max(mf, nf))
    runs = [_kernel_runs(s) for s in scales if s > 0]
    d_runs = _device.to_device(np.concatenate(runs).astype(np.int32)) if runs else None
    scratch = torch.empty((mf, nf + 1), dtype=torch.int64, device="cuda")
    out = torch.empty((T, mf, nf), dtype=torch.float64, device="cuda")
    c_scales = (_lib.c_int * T)(*scales)
    _lib.call("b200_probability", F.data_ptr(), _device.dtype_code(F.dtype), plane_stride, T, mf, nf,
              threshold_cmp, int(nan_exceeds), c_scales, _device.ptr(d_runs), scratch.data_ptr(), out.data_ptr(),
              _device.stream_ptr())
    return out if on_device else _device.to_host(out)


def _fail_as_the_reference(F, threshold):
    """What the reference's first two array operations do with an extrapolator's None or
    (field, displacement) tuple: they raise."""
    if isinstance(F, tuple):
        F = tuple(_device.to_host(x) if _device.is_device_tensor(x) else x for x in F)
    nanmask = np.isnan(F)
    F[nanmask] = threshold - 1
    raise TypeError(f"the extrapolator returned {type(F).__name__}, not a field")


def _threshold_rule(dtype, threshold):
    """(t, nan_exceeds): a valid pixel v exceeds when (double)v >= t, a NaN pixel when nan_exceeds.
    The reference sets NaN pixels to `threshold - 1` in the field's dtype, then compares the field
    with `threshold` in NumPy's result dtype (float32 for a float32 field and a Python scalar)."""
    dt = np.float32 if dtype == torch.float32 else np.float64
    fill = np.zeros(1, dtype=dt)
    fill[0] = threshold - 1
    nan_exceeds = bool((fill >= threshold)[0])
    return _compare.comparison_threshold(dt, threshold, "lagrangian_probability")[0], nan_exceeds


def _scales(timesteps, slope, side):
    """int(t * slope) of every lead, with the reference's failure for a negative diameter."""
    scales = []
    for t in timesteps:
        s = int(t * slope)
        if s < 0:
            raise ValueError("negative dimensions are not allowed")  # numpy, building the kernel
        if s > _MAX_SCALE or side + s >= 1 << 31:
            raise NotImplementedError("pysteps_b200 lagrangian_probability: kernel diameters above 2^24 px are "
                                      "not supported")
        scales.append(s)
    return scales


def _kernel_runs(s):
    """(s, 2) int64: first and last column of every row of the reference's kernel of diameter s > 0,
    an s x s block of ones for s < 5, else the disk (a - mid)^2 + (b - mid)^2 <= mid^2 on the s x s
    grid, mid = max(s // 2, 1) (truncated at column s - 1 for even s).  Exact integer square roots."""
    if s < 5:
        return np.tile(np.array([0, s - 1], dtype=np.int64), (s, 1))
    mid = max(s // 2, 1)
    a = np.arange(s, dtype=np.int64)
    d = mid * mid - (a - mid) ** 2
    r = np.floor(np.sqrt(d.astype(np.float64))).astype(np.int64)
    r += (r + 1) ** 2 <= d  # the float square root is within one of the integer one
    r -= r * r > d
    return np.stack([np.maximum(mid - r, 0), np.minimum(mid + r, s - 1)], axis=1)
