"""Mirror of pysteps/verification/interface.py for the verification scores built on the device.

``get_method(name, type)`` takes the reference's names and types, case-insensitive, with the same
``None`` handling and the same ValueError texts.  The probabilistic scores ("crps", "reldiag", "roc")
and the rank histogram ("rankhist", type "ensemble") are probscores.py and ensscores.py here.  The
other names the reference knows (the deterministic scores, "ens_skill", "ens_spread") are not
dispatched by ``get_method``: they raise NotImplementedError naming the device function to call
instead where there is one (``det_cat_fct``, ``det_cont_fct``, ``fss``, ``ensemble_skill``,
``ensemble_spread``), and pointing to pysteps.verification otherwise.  pysteps keeps no registry dict
for these scores, so ``pysteps_b200.register()`` does not publish them: import them from here.
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
_DEVICE_FUNCTION = dict({n: "detcatscores.det_cat_fct" for n in ensscores.CATEGORICAL},
                        **{n: "detcontscores.det_cont_fct" for n in ensscores.CONTINUOUS
                           if n not in ("corr_s", "scatter")},
                        fss="spatialscores.fss", ens_skill="ensscores.ensemble_skill",
                        ens_spread="ensscores.ensemble_spread")


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
        if name in _DEVICE_FUNCTION:
            raise NotImplementedError(f"pysteps_b200: get_method does not dispatch the {type} score {name!r}; call "
                                      f"pysteps_b200.verification.{_DEVICE_FUNCTION[name]}, or "
                                      "pysteps.verification.get_method for the reference")
        raise NotImplementedError(f"pysteps_b200: the {type} score {name!r} is not built on the device; "
                                  "use pysteps.verification.get_method")
    raise ValueError("unknown %s method %s" % (type, name))
