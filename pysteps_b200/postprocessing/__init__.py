"""B200 mirror of ``pysteps.postprocessing`` for the ensemble statistics, whose reductions run on the device."""
from . import ensemblestats  # noqa: F401
from .interface import get_method  # noqa: F401
