"""Mirror of pysteps/motion/interface.py:36-111 for the B200 motion methods.

Same ``get_method(name)`` contract: case-insensitive names, ``None`` -> a callable that
returns a zero field, unknown names -> ValueError, "brox"/"clg" -> NotImplementedError
(pysteps/motion/interface.py:97-111).  "proesmans" is built but opt-in until verified on
hardware (see motion/proesmans.py); "constant" is motion/constant.py; "darts" is motion/darts.py;
farneback is not provided.
"""
import numpy as np

from .lucaskanade import dense_lucaskanade

_methods = dict()
_methods["lk"] = dense_lucaskanade
_methods["lucaskanade"] = dense_lucaskanade
_methods["lk_b200"] = dense_lucaskanade
_methods[None] = lambda precip, *args, **kw: np.zeros((2, precip.shape[1], precip.shape[2]))
try:
    from .vet import vet
    _methods["vet"] = vet
    _methods["vet_b200"] = vet
except ImportError:  # VET not built yet
    pass


from .proesmans import proesmans  # noqa: E402

_methods["proesmans"] = proesmans
_methods["proesmans_b200"] = proesmans

from .constant import constant  # noqa: E402

_methods["constant"] = constant
_methods["constant_b200"] = constant

from .darts import DARTS  # noqa: E402

_methods["darts"] = DARTS
_methods["darts_b200"] = DARTS


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
