"""B200 mirror of ``pysteps.postprocessing`` for the ensemble statistics and probability matching, which
run on the device."""
from . import ensemblestats, probmatching  # noqa: F401
from .interface import get_method  # noqa: F401
