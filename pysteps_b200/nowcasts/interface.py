"""Mirror of pysteps/nowcasts/interface.py:44-110 for the B200 nowcast models.

Same ``get_method(name)`` contract: case-insensitive names, TypeError for a name that is not a
string, ValueError for an unknown one.  "lagrangian_probability" (alias "probability") is
nowcasts/lagrangian_probability.py, "extrapolation" (alias "lagrangian") nowcasts/extrapolation.py
and "eulerian" the Eulerian persistence of extrapolation/interface.py; the other models of the
reference are not provided.
"""
from ..extrapolation import interface as _extrapolation
from ..interface import with_b200_names
from . import extrapolation, lagrangian_probability

PROVIDED = {"lagrangian_probability": lagrangian_probability.forecast, "probability": lagrangian_probability.forecast,
            "extrapolation": extrapolation.forecast, "lagrangian": extrapolation.forecast}

_nowcast_methods = with_b200_names(PROVIDED)
_nowcast_methods["eulerian"] = _extrapolation.eulerian_persistence


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
