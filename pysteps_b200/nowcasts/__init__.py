"""B200 mirror of ``pysteps.nowcasts`` for the nowcast models whose work runs on the device."""
from . import extrapolation, lagrangian_probability  # noqa: F401
from .interface import get_method  # noqa: F401
