"""Mirror of pysteps/extrapolation/interface.py:41-145 with the B200
semi-Lagrangian scheme behind the same ``get_method(name)`` contract."""
import numpy as np

from ..interface import with_b200_names
from . import semilagrangian


def eulerian_persistence(precip, velocity, timesteps, outval=np.nan, **kwargs):
    """Eulerian persistence (pysteps/extrapolation/interface.py:41-93): the input field
    replicated once per timestep.  Trivial replication; no kernel involved."""
    del velocity, outval
    if isinstance(timesteps, int):
        num_timesteps = timesteps
    else:
        num_timesteps = len(timesteps)
    return_displacement = kwargs.get("return_displacement", False)
    extrapolated_precip = np.repeat(precip[np.newaxis, :, :], num_timesteps, axis=0)
    if not return_displacement:
        return extrapolated_precip
    return extrapolated_precip, np.zeros((2,) + extrapolated_precip.shape)


def _do_nothing(precip, velocity, timesteps, outval=np.nan, **kwargs):
    del precip, velocity, timesteps, outval, kwargs
    return None


PROVIDED = {"semilagrangian": semilagrangian.extrapolate}

_extrapolation_methods = with_b200_names(PROVIDED)
_extrapolation_methods["eulerian"] = eulerian_persistence
_extrapolation_methods[None] = _do_nothing
_extrapolation_methods["none"] = _do_nothing


def get_method(name):
    """Same lookup rules as pysteps/extrapolation/interface.py:114-145."""
    if isinstance(name, str):
        name = name.lower()
    try:
        return _extrapolation_methods[name]
    except KeyError:
        raise ValueError(
            "Unknown method {}\n".format(name)
            + "The available methods are:"
            + str(list(_extrapolation_methods.keys()))
        ) from None
