"""ctypes binding of ``libpysteps_b200.so`` (the C ABI declared in
``include/pysteps_b200.h``).

There is NO fallback: if the shared library is missing or a call fails, the
product path raises.  Build it with ``python -c "import __graft_entry__ as g;
g.build()"`` or ``make -C pysteps_b200/csrc``.
"""
import ctypes
import os
import re
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpysteps_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "pysteps_b200.h")

F32, F64 = 0, 1
MODE_CONSTANT, MODE_NEAREST = 0, 1
LAYOUT_PLANAR, LAYOUT_INTERLEAVED = 0, 1
LK_MAX_LEVELS = 16  # B200_LK_MAX_LEVELS: entries of b200_lk_pyramid_layout's level arrays
VERIF_MAX_MEMBERS, VERIF_MAX_BINS = 512, 2048  # B200_VERIF_MAX_MEMBERS / _MAX_BINS
FSS_GROUP = 16  # B200_FSS_GROUP: fields per group of b200_fss_sums
# B200_MOM_*: the element-wise operations of b200_verif_cont_moments that overflowed (OVER) or made a NaN (INV)
(MOM_SUB_RES_OVER, MOM_SUB_RES_INV, MOM_ADD_SUM_OVER, MOM_ADD_SUM_INV, MOM_SQ_RES_OVER, MOM_SQ_SUM_OVER,
 MOM_SUB_OBS_OVER, MOM_SUB_OBS_INV, MOM_SUB_PRED_OVER, MOM_SUB_PRED_INV, MOM_MUL_OVER, MOM_MUL_INV, MOM_SQ_VOBS_OVER,
 MOM_SQ_VPRED_OVER) = (1 << i for i in range(14))

_lib = None
_lock = threading.Lock()

c_void_p, c_int, c_i64, c_double = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double
c_dp = ctypes.POINTER(ctypes.c_double)

# name -> (restype, argtypes); must list every function declared in the header
_SIGNATURES = {
    "b200_version": (c_int, []),
    "b200_last_error": (ctypes.c_char_p, []),
    "b200_launch_count": (ctypes.c_longlong, []),
    "b200_device_info": (c_int, [ctypes.POINTER(c_int)] * 3 + [ctypes.c_char_p, c_int]),
    "b200_sl_extrapolate": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_dp, c_int, c_double,
                                    c_int, c_double, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p, c_void_p, c_void_p]),
    "b200_sl_extrapolate_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_dp, c_int, c_double,
                                         c_int, c_double, c_int, c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_sl_extrapolate_rows_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_dp, c_int, c_double, c_double, c_int,
                                             c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                             c_void_p, c_void_p]),
    "b200_sl_interleave_velocity": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_sl_trajectories": (c_int, [c_void_p, c_void_p, c_void_p, c_dp, c_int, c_double, c_int, c_int, c_int,
                                     c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_spline_prepare": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_dp,
                                    c_dp, c_dp, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_spline_sample": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                   c_int, c_double, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b200_proesmans_scale": (c_int, [c_void_p, c_int, ctypes.c_int64, c_double, c_double, c_int, c_void_p, c_void_p]),
    "b200_gaussian_filter": (c_int, [c_void_p, c_int, c_int, c_dp, c_int, c_void_p, c_void_p]),
    "b200_proesmans_field": (c_int, [c_void_p, c_int, c_int, c_double, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_bps_perturb_velocity": (c_int, [c_void_p, c_int, c_int, c_int, c_double, c_double, c_double,
                                          c_int, c_void_p, c_void_p, c_void_p]),
    "b200_sl_extrapolate_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_dp, c_int,
                                         c_double, c_int, c_double, c_int, c_int, c_int, c_int,
                                         c_int, c_void_p, c_void_p]),
    "b200_mask_invalid": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_morph_opening": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                   c_void_p, c_void_p]),
    "b200_masked_minmax": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                   c_void_p]),
    "b200_quantise_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p]),
    "b200_fill_f64": (c_int, [c_void_p, c_i64, c_double, c_void_p]),
    "b200_pyr_down_u8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200_scharr_i16": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200_min_eig": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200_good_features": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_double,
                                   c_void_p, c_void_p, c_void_p]),
    "b200_lk_pyramid_layout": (c_int, [c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int),
                                       ctypes.POINTER(c_i64), ctypes.POINTER(c_int),
                                       ctypes.POINTER(c_int), ctypes.POINTER(c_i64)]),
    "b200_sl_step_batched": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_double, c_void_p, c_int,
                                     c_void_p, c_double, c_double, c_double, c_int, c_void_p, c_void_p, c_void_p,
                                     c_void_p]),
    "b200_lk_frontend": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_lk_build_pyramid": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p]),
    "b200_lk_track": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                              c_double, c_double, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                              c_void_p]),
    "b200_lk_compact_tracks": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                       c_void_p, c_int, c_void_p]),
    "b200_detect_outliers": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_double, c_int, c_void_p,
                                     c_void_p]),
    "b200_detect_outliers_global": (c_int, [c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p]),
    "b200_idw_fill_all": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_double, c_double, c_double,
                                  c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "b200_kdtree_build": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_compact_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "b200_decluster": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_double, c_int, c_void_p, c_void_p,
                               c_void_p, c_void_p]),
    "b200_idw_fill": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_double,
                              c_double, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200_idw_plan": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200_idw_fill_planned": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_double, c_double, c_void_p,
                                      c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_idw_fill_ckdtree": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_double,
                                      c_double, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "b200_vet_cost": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                              ctypes.c_float, c_int, c_void_p, c_void_p]),
    "b200_vet_value_and_gradient": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int,
                                            ctypes.c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_vet_level_images": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                      c_void_p, c_void_p, c_void_p]),
    "b200_vet_warp": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                              c_void_p]),
    "b200_zoom_bilinear": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_field_stats": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_void_p]),
    "b200_constant_scratch_bytes": (c_int, [c_int, c_int, ctypes.POINTER(c_i64)]),
    "b200_constant_eval": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_double, c_void_p,
                                   c_void_p, c_void_p]),
    "b200_darts_spectrum": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                    c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_darts_normal": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double, c_void_p,
                                  c_void_p, c_void_p, c_void_p]),
    "b200_darts_synthesize": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                      c_void_p]),
    "b200_probability": (c_int, [c_void_p, c_int, c_i64, c_int, c_int, c_int, c_double, c_int,
                                 ctypes.POINTER(c_int), c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_ensemble_mean": (c_int, [c_void_p, c_int, c_int, c_i64, c_int, c_int, c_double, c_void_p, c_void_p,
                                   c_void_p]),
    "b200_ensemble_excprob": (c_int, [c_void_p, c_int, c_int, c_i64, c_dp, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p]),
    "b200_ensemble_band_mask": (c_int, [c_void_p, c_int, c_int, c_i64, c_double, c_void_p, c_void_p, c_void_p]),
    "b200_ensemble_band_match": (c_int, [c_void_p, c_int, c_int, c_i64, c_void_p, c_void_p, c_i64, c_void_p,
                                         c_void_p]),
    "b200_blend_transform": (c_int, [c_void_p, c_void_p, c_int, c_i64, c_int, c_double, c_double, c_double,
                                     c_void_p, c_void_p, c_i64, c_void_p, c_void_p]),
    "b200_blend_unit": (c_int, [c_void_p, c_void_p, c_int, c_i64, c_int, c_double, c_double, c_void_p]),
    "b200_blend_scatter": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_i64, c_void_p]),
    "b200_blend_linear": (c_int, [c_void_p, c_int, c_void_p, c_i64, c_void_p, c_int, c_void_p, c_i64, c_void_p,
                                  c_int, c_int, c_i64, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "b200_blend_scratch_bytes": (c_int, [c_i64, ctypes.POINTER(c_i64)]),
    "b200_blend_salient": (c_int, [c_void_p, c_int, c_void_p, c_i64, c_void_p, c_int, c_void_p, c_i64, c_void_p,
                                   c_int, c_int, c_i64, c_int, c_double, c_double, c_double, c_double, c_int,
                                   c_void_p, c_i64, c_void_p]),
    "b200_dense_rank": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "b200_pairwise_sum": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b200_verif_crps": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_i64, c_void_p, c_void_p, c_void_p]),
    "b200_verif_rankhist": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_i64, c_int, c_double, c_double,
                                    c_double, c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_verif_rankhist_ties": (c_int, [c_void_p, c_i64, c_void_p, c_int, c_void_p, c_void_p]),
    "b200_verif_reldiag": (c_int, [c_void_p, c_int, c_void_p, c_int, c_i64, c_dp, c_int, c_double, c_void_p,
                                   c_void_p, c_void_p, c_void_p]),
    "b200_verif_roc": (c_int, [c_void_p, c_int, c_void_p, c_int, c_i64, c_dp, c_int, c_double, c_void_p,
                               c_void_p]),
    "b200_verif_contab": (c_int, [c_void_p, c_int, c_void_p, c_int, c_double, c_double, ctypes.POINTER(c_i64),
                                  ctypes.POINTER(c_i64), c_int, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64), c_int,
                                  c_void_p, c_void_p]),
    "b200_verif_cont_moments": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_double, c_double,
                                        ctypes.POINTER(c_i64), ctypes.POINTER(c_i64), c_int, ctypes.POINTER(c_i64),
                                        ctypes.POINTER(c_i64), c_int, c_i64, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p]),
    "b200_fss_fractions": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_double, c_double, c_int, c_void_p,
                                   c_void_p]),
    "b200_fss_sums": (c_int, [c_void_p, c_i64, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_pm_scratch_bytes": (c_int, [c_i64, ctypes.POINTER(c_i64)]),
    "b200_pm_match_stats": (c_int, [c_void_p, c_int, c_void_p, c_i64, c_void_p, c_int, c_i64, c_void_p, c_void_p,
                                    c_i64, c_void_p]),
    "b200_pm_match": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_i64, c_void_p, c_i64, c_i64, c_int, c_i64,
                              c_i64, c_double, c_void_p, c_void_p, c_i64, c_void_p]),
    "b200_pm_resample_nan": (c_int, [c_void_p, c_int, c_void_p, c_int, c_i64, c_void_p, c_void_p]),
    "b200_pm_resample": (c_int, [c_void_p, c_int, c_void_p, c_int, c_i64, c_i64, c_void_p, c_void_p, c_int, c_void_p,
                                 c_i64, c_void_p]),
}


def header_symbols():
    """Names of all functions declared in include/pysteps_b200.h."""
    with open(HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def load():
    """Load the CUDA library; raise RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"pysteps_b200: CUDA library not built ({LIB_PATH} missing). "
                    "Run `make -C pysteps_b200/csrc` (needs nvcc, sm_90a). "
                    "There is no CPU fallback.")
            lib = ctypes.CDLL(LIB_PATH)
            for name, (res, args) in _SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        msg = load().b200_last_error()
        raise RuntimeError(f"pysteps_b200 CUDA call failed (code {rc}): "
                           f"{msg.decode(errors='replace') if msg else ''}")


# --- optional tracing: CUDA events around every C-ABI call (bench.py / profiling) ---------
_trace = None


class Trace:
    """Records (name, start_event, end_event) for each traced C-ABI call on the current
    torch stream.  ``summary()`` synchronises and returns {name: [ms, ...]}."""

    def __init__(self, only=None):
        """only: trace just these entry points (two CUDA events per traced call cost ~15 us of host
        time; a timed region traces the one kernel it rates, the per-stage table comes from
        untimed steps)."""
        self.records = []
        self.only = None if only is None else frozenset(only)

    def __enter__(self):
        global _trace
        self._prev = _trace
        _trace = self
        return self

    def __exit__(self, *exc):
        global _trace
        _trace = self._prev

    def summary(self):
        import torch
        torch.cuda.synchronize()
        out = {}
        for name, s, e in self.records:
            out.setdefault(name, []).append(s.elapsed_time(e))
        return out


def call(name, *args):
    """Invoke a C-ABI function by name, raising on failure; traced when a Trace is active."""
    fn = getattr(load(), name)
    tr = _trace
    if tr is None or (tr.only is not None and name not in tr.only):
        check(fn(*args))
        return
    import torch
    s = torch.cuda.Event(enable_timing=True)
    e = torch.cuda.Event(enable_timing=True)
    s.record()
    rc = fn(*args)
    e.record()
    tr.records.append((name, s, e))
    check(rc)
