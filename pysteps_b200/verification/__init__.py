"""B200 mirror of ``pysteps.verification`` for the scores whose accumulation runs on the device: CRPS,
the reliability diagram and the ROC curve (probscores), and the rank histogram (ensscores)."""
from . import ensscores  # noqa: F401
from . import probscores  # noqa: F401
from .interface import get_method  # noqa: F401
