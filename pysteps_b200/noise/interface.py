"""Mirror of pysteps/noise/interface.py:24-104 for the one method on the advection path:
``get_method("bps")`` -> (initialize_bps, generate_bps).  The precipitation noise generators
(parametric, nonparametric, ssft, nested) are FFT filters outside this path and are not
provided."""
from ..interface import with_b200_names
from . import motion

PROVIDED = {"bps": (motion.initialize_bps, motion.generate_bps)}

_noise_methods = with_b200_names(PROVIDED)


def get_method(name):
    """Same lookup rules as pysteps/noise/interface.py:48-104."""
    if isinstance(name, str):
        name = name.lower()
    else:
        raise TypeError(
            "Only strings supported for the method's names.\n"
            + "Available names:"
            + str(list(_noise_methods.keys()))
        ) from None
    try:
        return _noise_methods[name]
    except KeyError:
        raise ValueError(
            "Unknown method {}\n".format(name)
            + "The available methods are:"
            + str(list(_noise_methods.keys()))
        ) from None
