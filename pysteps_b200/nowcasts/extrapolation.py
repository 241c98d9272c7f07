"""B200 extrapolation nowcast -- drop-in for ``pysteps.nowcasts.extrapolation.forecast``
(pysteps/nowcasts/extrapolation.py).

The input checks, ``allow_nonfinite_values`` rule, ``measure_time`` prints and return are the
reference's.  The semi-Lagrangian names call the device extrapolator with device tensors, and the
field's finiteness is a device reduction, so a CUDA-tensor precip never leaves HBM.  NumPy input
returns NumPy; a CUDA-tensor precip returns a CUDA tensor.  Other extrapolators (``"eulerian"``, a
plug-in) are called with the caller's arrays as the reference calls them.
"""
import time

import numpy as np

from .. import _device
from ..extrapolation import interface as _extrapolation
from ..extrapolation import semilagrangian as _sl
from ..noise import motion as _bps


def check_inputs(precip, velocity, timesteps):
    """nowcasts/extrapolation.py:_check_inputs, shared by every nowcast of this package."""
    if precip.ndim != 2:
        raise ValueError("The input precipitation must be a " "two-dimensional array")
    if velocity.ndim != 3:
        raise ValueError("Input velocity must be a three-dimensional array")
    if precip.shape != velocity.shape[1:3]:
        raise ValueError(
            "Dimension mismatch between "
            "input precipitation and velocity: "
            + "shape(precip)=%s, shape(velocity)=%s"
            % (str(precip.shape), str(velocity.shape))
        )
    if isinstance(timesteps, list) and not sorted(timesteps) == timesteps:
        raise ValueError("timesteps is not in ascending order")


def device_velocity(velocity):
    """The velocity as the device extrapolator takes it without a copy back to the host."""
    if _device.is_device_tensor(velocity) or isinstance(velocity, _bps.PerturbedVelocity):
        return velocity
    return _sl._field_tensor(velocity)


def forecast(precip, velocity, timesteps, extrap_method="semilagrangian", extrap_kwargs=None, measure_time=False):
    """Same contract as the reference: precip (m, n), velocity (2, m, n); returns the (T, m, n)
    extrapolated fields, and the computation time when `measure_time`."""
    check_inputs(precip, velocity, timesteps)

    if extrap_kwargs is None:
        extrap_kwargs = dict()
    else:
        extrap_kwargs = extrap_kwargs.copy()

    _device.require_cuda()
    on_device = _device.is_device_tensor(precip)
    d_precip = _sl._field_tensor(precip)
    # np.any(~np.isfinite(precip)) as a device reduction
    extrap_kwargs["allow_nonfinite_values"] = bool(_sl._Stats(d_precip).get()[0][0] > 0)

    if measure_time:
        print(
            "Computing extrapolation nowcast from a "
            f"{precip.shape[0]:d}x{precip.shape[1]:d} input grid... ",
            end="",
        )

    if measure_time:
        start_time = time.time()

    extrapolation_method = _extrapolation.get_method(extrap_method)

    if extrapolation_method is _sl.extrapolate:
        precip_forecast = extrapolation_method(d_precip, device_velocity(velocity), timesteps, **extrap_kwargs)
        if not on_device:
            precip_forecast = _to_host(precip_forecast)
    else:
        args = (precip, velocity) if not on_device else (_device.to_host(precip), _to_host(velocity))
        precip_forecast = extrapolation_method(*args, timesteps, **extrap_kwargs)
        if on_device:
            precip_forecast = _to_device(precip_forecast)

    if measure_time:
        computation_time = time.time() - start_time
        print(f"{computation_time:.2f} seconds.")

    if measure_time:
        return precip_forecast, computation_time
    else:
        return precip_forecast


def _to_host(x):
    if isinstance(x, tuple):
        return tuple(_to_host(v) for v in x)
    return _device.to_host(x) if _device.is_device_tensor(x) else x


def _to_device(x):
    if isinstance(x, tuple):
        return tuple(_to_device(v) for v in x)
    return _device.to_device(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
