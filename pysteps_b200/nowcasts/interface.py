"""Mirror of pysteps/nowcasts/interface.py:44-110 for the B200 nowcast models.

Same ``get_method(name)`` contract: case-insensitive names, TypeError for a name that is not a
string, ValueError for an unknown one.  "lagrangian_probability" (alias "probability") is
nowcasts/lagrangian_probability.py, "extrapolation" (alias "lagrangian") nowcasts/extrapolation.py
and "eulerian" the Eulerian persistence of extrapolation/interface.py; the other models of the
reference are not provided.
"""
from ..extrapolation import interface as _extrapolation
from . import extrapolation, lagrangian_probability

_nowcast_methods = dict()
_nowcast_methods["lagrangian_probability"] = lagrangian_probability.forecast
_nowcast_methods["lagrangian_probability_b200"] = lagrangian_probability.forecast
_nowcast_methods["probability"] = lagrangian_probability.forecast
_nowcast_methods["probability_b200"] = lagrangian_probability.forecast
_nowcast_methods["eulerian"] = _extrapolation.eulerian_persistence
_nowcast_methods["extrapolation"] = extrapolation.forecast
_nowcast_methods["extrapolation_b200"] = extrapolation.forecast
_nowcast_methods["lagrangian"] = extrapolation.forecast
_nowcast_methods["lagrangian_b200"] = extrapolation.forecast


def get_method(name):
    if isinstance(name, str):
        name = name.lower()
    else:
        raise TypeError(
            "Only strings supported for the method's names.\n"
            + "Available names:"
            + str(list(_nowcast_methods.keys()))
        ) from None
    try:
        return _nowcast_methods[name]
    except KeyError:
        raise ValueError(
            "Unknown nowcasting method {}\n".format(name)
            + "The available methods are:"
            + str(list(_nowcast_methods.keys()))
        ) from None
