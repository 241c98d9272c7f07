"""Mirror of pysteps/postprocessing/interface.py:187-266 for the B200 ensemble statistics.

Same ``get_method(name, method_type)`` contract: case-insensitive names and types, TypeError for a
name or type that is not a string, ValueError for an unknown one.  The "ensemblestats" methods are
postprocessing/ensemblestats.py under the reference's names and with a "_b200" suffix; there are no
"diagnostics" methods, as in the reference without plugins.
"""
from ..interface import with_b200_names
from . import ensemblestats

PROVIDED = {"mean": ensemblestats.mean, "excprob": ensemblestats.excprob, "banddepth": ensemblestats.banddepth}

_diagnostics_methods = dict()

_ensemblestats_methods = with_b200_names(PROVIDED)


def get_method(name, method_type):
    if isinstance(method_type, str):
        method_type = method_type.lower()
    else:
        raise TypeError(
            "Only strings supported for for the method_type"
            + " argument\n"
            + "The available types are: 'diagnostics', 'ensemblestats'"
        ) from None

    if isinstance(name, str):
        name = name.lower()
    else:
        raise TypeError(
            "Only strings supported for the method's names.\n"
            + "\nAvailable diagnostics names:"
            + str(list(_diagnostics_methods.keys()))
            + "\nAvailable ensemblestats names:"
            + str(list(_ensemblestats_methods.keys()))
        ) from None

    if method_type == "diagnostics":
        methods_dict = _diagnostics_methods
    elif method_type == "ensemblestats":
        methods_dict = _ensemblestats_methods
    else:
        raise ValueError(
            "Unknown method type {}\n".format(method_type)
            + "The available types are: 'diagnostics', 'ensemblestats'"
        ) from None

    try:
        return methods_dict[name]
    except KeyError:
        raise ValueError(
            "Unknown {} method {}\n".format(method_type, name)
            + "The available methods are:"
            + str(list(methods_dict.keys()))
        ) from None
