"""Mirror of pysteps/verification/interface.py for the verification scores built on the device.

``get_method(name, type)`` takes the reference's names and types, case-insensitive, with the same
``None`` handling and the same ValueError texts.  The probabilistic scores ("crps", "reldiag", "roc")
and the rank histogram ("rankhist", type "ensemble") are probscores.py and ensscores.py here; the
other names the reference knows (the deterministic scores, "ens_skill", "ens_spread") raise
NotImplementedError and point to pysteps.verification.  pysteps keeps no registry dict for these
scores, so ``pysteps_b200.register()`` does not publish them: import them from here.
"""
from . import ensscores, probscores

_DETERMINISTIC = ("acc", "bias", "csi", "f1", "fa", "far", "gss", "hk", "hss", "mcc", "pod", "sedi",
                  "beta", "beta1", "beta2", "corr_p", "corr_s", "drmse", "mae", "mse", "me", "nmse",
                  "rmse", "rv", "scatter", "binary_mse", "fss", "sal")

_PROVIDED = {
    "ensemble": {"rankhist": ensscores.rankhist},
    "probabilistic": {"crps": probscores.CRPS, "reldiag": probscores.reldiag, "roc": probscores.ROC_curve},
}
_NOT_BUILT = {"deterministic": _DETERMINISTIC, "ensemble": ("ens_skill", "ens_spread")}


def get_method(name, type="deterministic"):
    """The device callable of the verification score `name` of `type` ("deterministic",
    "ensemble" or "probabilistic")."""
    name = "none" if name is None else name
    type = "none" if type is None else type
    name, type = name.lower(), type.lower()
    if type not in ("deterministic", "ensemble", "probabilistic"):
        raise ValueError("unknown type %s" % name)
    if name in _PROVIDED.get(type, {}):
        return _PROVIDED[type][name]
    if name in _NOT_BUILT.get(type, ()):
        raise NotImplementedError(f"pysteps_b200: the {type} score {name!r} is not built on the device; "
                                  "use pysteps.verification.get_method")
    raise ValueError("unknown %s method %s" % (type, name))
