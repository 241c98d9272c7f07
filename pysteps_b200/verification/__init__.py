"""B200 mirror of ``pysteps.verification`` for the scores whose accumulation runs on the device: the
contingency-table scores (detcatscores), the online continuous scores (detcontscores), the fractions
skill score and its intensity-scale table (spatialscores), CRPS, the reliability diagram and the ROC
curve (probscores), and the rank histogram and the ensemble skill and spread (ensscores).  As in
pysteps, the functions are also exported here: ``pysteps_b200.verification.fss(...)``,
``det_cat_fct(...)``."""
from . import detcatscores, detcontscores, ensscores, probscores, spatialscores  # noqa: F401
from .detcatscores import (det_cat_fct, det_cat_fct_accum, det_cat_fct_compute, det_cat_fct_init,  # noqa: F401
                           det_cat_fct_merge)
from .detcontscores import (det_cont_fct, det_cont_fct_accum, det_cont_fct_compute,  # noqa: F401
                            det_cont_fct_init, det_cont_fct_merge)
from .ensscores import (ensemble_skill, ensemble_spread, rankhist, rankhist_accum, rankhist_compute,  # noqa: F401
                        rankhist_init)
from .interface import get_method  # noqa: F401
from .probscores import (CRPS, CRPS_accum, CRPS_compute, CRPS_init, ROC_curve, ROC_curve_accum,  # noqa: F401
                         ROC_curve_compute, ROC_curve_init, reldiag, reldiag_accum, reldiag_compute,
                         reldiag_init)
from .spatialscores import (binary_mse, fss, fss_accum, fss_compute, fss_init, fss_merge,  # noqa: F401
                            intensity_scale, intensity_scale_accum, intensity_scale_compute, intensity_scale_init,
                            intensity_scale_merge, sal)
