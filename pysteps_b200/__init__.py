"""pysteps_b200 -- CUDA-native (H100, sm_90a) advection hot path for pysteps.

Drop-in replacements, behind pysteps' own ``get_method()`` registries, for
  * ``pysteps.extrapolation.semilagrangian.extrapolate``
  * ``pysteps.motion.lucaskanade.dense_lucaskanade``
  * ``pysteps.motion.vet.vet``
  * ``pysteps.noise.motion.initialize_bps`` / ``generate_bps`` (fused into the advection call)
  * ``pysteps.nowcasts.lagrangian_probability.forecast`` and ``pysteps.nowcasts.extrapolation.forecast``
  * ``pysteps.postprocessing.ensemblestats.mean`` / ``excprob`` / ``banddepth``
  * ``pysteps.blending.linear_blending.forecast`` (linear and salient blending)
and, reached as ``pysteps_b200.verification`` (pysteps keeps no registry for them), the
  * ``pysteps.verification`` scores ``CRPS``, ``reldiag``, ``ROC_curve`` and ``rankhist``
Host code is Python; every array operation is a hand-written CUDA kernel in
``libpysteps_b200.so`` reached through ctypes (``include/pysteps_b200.h``).
There is no CPU fallback: without the built library and a GPU, calls raise.
"""
__version__ = "0.1.0"

from . import blending  # noqa: F401
from . import extrapolation  # noqa: F401
from . import motion  # noqa: F401
from . import noise  # noqa: F401
from . import nowcasts  # noqa: F401
from . import postprocessing  # noqa: F401
from . import verification  # noqa: F401
from .interface import register  # noqa: F401
