"""Mirror of pysteps/motion/interface.py:36-111 for the B200 motion methods.

Same ``get_method(name)`` contract: case-insensitive names, ``None`` -> a callable that
returns a zero field, unknown names -> ValueError, "brox"/"clg" -> NotImplementedError
(pysteps/motion/interface.py:97-111).  "proesmans" is built but opt-in until verified on
hardware (see motion/proesmans.py); "constant" is motion/constant.py; "darts" is motion/darts.py;
farneback is not provided.
"""
import numpy as np

from ..interface import with_b200_names
from .constant import constant
from .darts import DARTS
from .lucaskanade import dense_lucaskanade
from .proesmans import proesmans
from .vet import vet

PROVIDED = {"lk": dense_lucaskanade, "lucaskanade": dense_lucaskanade, "vet": vet, "proesmans": proesmans,
            "constant": constant, "darts": DARTS}

_methods = with_b200_names(PROVIDED)
_methods[None] = lambda precip, *args, **kw: np.zeros((2, precip.shape[1], precip.shape[2]))


def get_method(name):
    if isinstance(name, str):
        name = name.lower()
    if name in ["brox", "clg"]:
        raise NotImplementedError("Method {} not implemented".format(name))
    try:
        return _methods[name]
    except KeyError:
        raise ValueError(
            "Unknown method {}\n".format(name)
            + "The available methods are:"
            + str(list(_methods.keys()))
        ) from None
