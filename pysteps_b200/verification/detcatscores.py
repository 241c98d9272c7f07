"""B200 categorical verification scores -- drop-in for ``pysteps.verification.detcatscores``:
``det_cat_fct`` and its ``det_cat_fct_init`` / ``_accum`` / ``_merge`` / ``_compute`` steps.

``det_cat_fct_accum`` counts the contingency table on the device (csrc/detscores.cu): pred > thr and
obs > thr, compared in NumPy's dtype for each array, summed over the integration axes in place.  NaN
compares false, so a NaN pair counts as a "no" whatever the reference's docstring says, as in the
reference.  The dict is the reference's (int64 count arrays of the kept axes), so a table made by
pysteps can be accumulated here and finished by pysteps, and the reverse.  ``axis``: None integrates
everything, a negative axis alone integrates nothing, the negative entries of a mixed tuple are
dropped, as in the reference.  Inputs are NumPy arrays or CUDA tensors of float32 or float64 with at
most 4 dimensions and fewer than 2^31 elements; anything else raises NotImplementedError.
"""
import collections

import numpy as np
import torch

from .. import _device, _lib
from . import _inputs, _reduction


def det_cat_fct(pred, obs, thr, scores="", axis=None):
    """The categorical scores `scores` ("" for all of them) of pred against obs at threshold thr."""
    contab = det_cat_fct_init(thr, axis)
    det_cat_fct_accum(contab, pred, obs)
    return det_cat_fct_compute(contab, scores)


def axis_tuple(axis):
    """None, an iterable of axes as it is, or a single axis as a 1-tuple (the reference's dict value)"""
    if axis is None or (isinstance(axis, collections.abc.Iterable) and not isinstance(axis, int)):
        return axis
    return (axis,)


def det_cat_fct_init(thr, axis=None):
    """An empty contingency table for threshold thr, integrated over `axis`."""
    return {"thr": thr, "axis": axis_tuple(axis), "hits": None, "false_alarms": None, "misses": None,
            "correct_negatives": None}


def check_array(a, who, name):
    _inputs.check(a, who, name)
    if a.ndim > 4:
        raise NotImplementedError(f"pysteps_b200 {who}: {name} of more than 4 dimensions is not supported")
    _inputs.check_pixels(_inputs.pixels(a.shape), who)


def det_cat_fct_accum(contab, pred, obs):
    """Add the contingency counts of pred and obs to the table."""
    who = "det_cat_fct_accum"
    check_array(pred, who, "pred")
    check_array(obs, who, "obs")
    shape, oshape = tuple(int(s) for s in pred.shape), tuple(int(s) for s in obs.shape)
    if shape != oshape:
        raise ValueError("the shape of pred does not match the shape of obs %s!=%s" % (shape, oshape))
    nshape, axis = _reduction.kept_shape(shape, contab["axis"])
    thr = contab["thr"]
    thr_p = _inputs.threshold(_inputs.np_dtype(pred), thr, who)
    thr_o = _inputs.threshold(_inputs.np_dtype(obs), thr, who)
    keys = ("hits", "false_alarms", "misses", "correct_negatives")
    if contab["hits"] is None:
        for key in keys:
            contab[key] = np.zeros(nshape, dtype=int)
    elif contab["hits"].shape != nshape:
        raise ValueError("the shape of the input arrays does not match the shape of the contingency table %s!=%s"
                         % (nshape, contab["hits"].shape))
    eshape, eaxis = _reduction.effective(shape, axis)
    M = _inputs.pixels(nshape)
    if M * _inputs.pixels(eshape) == 0:
        return
    (ks, kst), (rs, rst) = _reduction.split_axes(eshape, eaxis)
    p = _inputs.to_device(pred, (-1,))
    o = _inputs.to_device(obs, (-1,))
    counts = torch.empty(4 * M, dtype=torch.int64, device="cuda")
    _lib.call("b200_verif_contab", p.data_ptr(), _device.dtype_code(p.dtype), o.data_ptr(),
              _device.dtype_code(o.dtype), thr_p, thr_o, *_reduction.c_axes(ks, kst), *_reduction.c_axes(rs, rst),
              counts.data_ptr(), _device.stream_ptr())
    c = _device.to_host(counts).reshape(4, M)
    for key, row in zip(keys, c):
        contab[key] += row.reshape(nshape)


def det_cat_fct_merge(contab_1, contab_2):
    """contab_1 with the counts of contab_2 added (a shallow copy: contab_1's arrays are updated in
    place, as in the reference)."""
    if contab_1["thr"] != contab_2["thr"]:
        raise ValueError("cannot merge: the thresholds are not same %s!=%s" % (contab_1["thr"], contab_2["thr"]))
    if contab_1["axis"] != contab_2["axis"]:
        raise ValueError("cannot merge: the axis are not same %s!=%s" % (contab_1["axis"], contab_2["axis"]))
    if contab_1["hits"] is None or contab_2["hits"] is None:
        raise ValueError("cannot merge: no data found")
    contab = contab_1.copy()
    for key in ("hits", "misses", "false_alarms", "correct_negatives"):
        contab[key] += contab_2[key]
    return contab


def score_names(scores):
    """a single name (a string or anything not iterable) as a 1-tuple"""
    if isinstance(scores, collections.abc.Iterable) and not isinstance(scores, str):
        return scores
    return (scores,)


def det_cat_fct_compute(contab, scores=""):
    """The scores of the table: "" for all, or any of acc, bias, csi, ets, f1, fa, far, gss, hk, hss, mcc,
    pod, sedi (case-insensitive); the keys are upper case."""
    H = 1.0 * contab["hits"]
    M = 1.0 * contab["misses"]
    F = 1.0 * contab["false_alarms"]
    R = 1.0 * contab["correct_negatives"]
    result = {}
    for score in score_names(scores):
        if score is None:
            continue
        name = score.lower()
        # every name evaluates the four rates first, as the reference does (and warns as often)
        pod = H / (H + M)
        far = F / (H + F)
        fa = F / (F + R)
        s = (H + M) / (H + M + F + R)
        if name in ("pod", ""):
            result["POD"] = pod
        if name in ("far", ""):
            result["FAR"] = far
        if name in ("fa", ""):
            result["FA"] = fa
        if name in ("acc", ""):
            result["ACC"] = (H + R) / (H + M + F + R)
        if name in ("csi", ""):
            result["CSI"] = H / (H + M + F)
        if name in ("bias", ""):
            result["BIAS"] = (H + F) / (H + M)
        if name in ("hss", ""):
            result["HSS"] = 2 * (H * R - F * M) / ((H + M) * (M + R) + (H + F) * (F + R))
        if name in ("hk", ""):
            result["HK"] = pod - fa
        if name in ("gss", "ets", ""):
            gss = (pod - fa) / ((1 - s * pod) / (1 - s) + fa * (1 - s) / s)
            result["ETS" if name == "ets" else "GSS"] = gss
        if name in ("sedi", ""):
            # the four logarithms are taken again for the denominator, as in the reference
            num = np.log(fa) - np.log(pod) + np.log(1 - pod) - np.log(1 - fa)
            result["SEDI"] = num / (np.log(fa) + np.log(pod) + np.log(1 - pod) + np.log(1 - fa))
        if name in ("mcc", ""):
            result["MCC"] = (H * R - F * M) / np.sqrt((H + F) * (H + M) * (R + F) * (R + M))
        if name in ("f1", ""):
            result["F1"] = 2 * H / (2 * H + F + M)
    return result
