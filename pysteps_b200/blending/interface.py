"""Mirror of pysteps/blending/interface.py for the B200 blending models.

Same ``get_method(name)`` contract: case-insensitive names, TypeError for a name that is not a
string, ValueError for an unknown one.  "linear_blending" and "salient_blending" (the same forecast
with saliency=True) are blending/linear_blending.py; "steps" and "pca_enkf" are not provided.
"""
from functools import partial

from ..interface import with_b200_names
from . import linear_blending

PROVIDED = {"linear_blending": linear_blending.forecast,
            "salient_blending": partial(linear_blending.forecast, saliency=True)}

_blending_methods = with_b200_names(PROVIDED)


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
