"""B200 mirror of ``pysteps.blending`` for the blending models whose work runs on the device."""
from . import linear_blending  # noqa: F401
from .interface import get_method  # noqa: F401
