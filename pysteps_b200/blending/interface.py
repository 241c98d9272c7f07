"""Mirror of pysteps/blending/interface.py for the B200 blending models.

Same ``get_method(name)`` contract: case-insensitive names, TypeError for a name that is not a
string, ValueError for an unknown one.  "linear_blending" and "salient_blending" (the same forecast
with saliency=True) are blending/linear_blending.py; "steps" and "pca_enkf" are not provided.
"""
from functools import partial

from . import linear_blending

_blending_methods = dict()
_blending_methods["linear_blending"] = linear_blending.forecast
_blending_methods["linear_blending_b200"] = linear_blending.forecast
_blending_methods["salient_blending"] = partial(linear_blending.forecast, saliency=True)
_blending_methods["salient_blending_b200"] = _blending_methods["salient_blending"]


def get_method(name):
    if isinstance(name, str):
        name = name.lower()
    else:
        raise TypeError(
            "Only strings supported for the method's names.\n"
            + "Available names:"
            + str(list(_blending_methods.keys()))
        ) from None

    try:
        return _blending_methods[name]
    except KeyError:
        raise ValueError(
            f"Unknown blending method {name}."
            "The available methods are: "
            f"{*list(_blending_methods.keys()),}"
        ) from None
