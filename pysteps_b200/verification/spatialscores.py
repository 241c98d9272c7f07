"""B200 spatial verification scores -- drop-in for the fractions skill score of
``pysteps.verification.spatialscores``: ``fss`` with its ``fss_init`` / ``_accum`` / ``_merge`` /
``_compute`` steps, and ``intensity_scale`` (with its steps) for the name "FSS".

``fss_accum`` thresholds both fields on the device (csrc/fss.cu): a non-finite value becomes thr - 1
rounded into the field's dtype (which for a large threshold in float32 can equal thr, as in the
reference), the indicator is X >= thr compared in NumPy's dtype, and for an integer size
s = int(scale) > 1 it is smoothed exactly as scipy.ndimage.uniform_filter(size=s, mode="constant")
smooths it.  The three sums of products are NumPy's pairwise sums over the plane, bit for bit.
The dict is the reference's, so dicts pass between the two packages both ways.

``binary_mse``, ``intensity_scale`` with "BMSE" and ``sal`` are not built on the device and raise
NotImplementedError.  Inputs are 2-D NumPy arrays or CUDA tensors of float32 or float64 with fewer
than 2^31 pixels.
"""
import collections

import numpy as np
import torch

from .. import _device, _lib
from . import _inputs


def fss(X_f, X_o, thr, scale):
    """The fractions skill score of X_f against X_o at threshold thr and spatial scale `scale`."""
    d = fss_init(thr, scale)
    fss_accum(d, X_f, X_o)
    return fss_compute(d)


def fss_init(thr, scale):
    """An empty FSS accumulator."""
    return dict(thr=thr, scale=scale, sum_fct_sq=0.0, sum_fct_obs=0.0, sum_obs_sq=0.0)


def filter_size(scale, who):
    """the size of the uniform filter fss_accum applies (1: none)"""
    if not scale > 1:
        return 1
    s = int(scale)
    if s >= 1 << 30:
        raise NotImplementedError(f"pysteps_b200 {who}: a scale of 2^30 or more is not supported")
    return s


def fractions(X, shape, thr, s, who):
    """the smoothed indicators of the 2-D fields of X (shape (nf, m, n)) as a (nf, m, n) float64 tensor"""
    dt = _inputs.np_dtype(X)
    t = _inputs.threshold(dt, thr, who)
    sub = float(np.asarray(thr - 1).astype(dt))  # stored into the field, so rounded to its dtype
    x = _inputs.to_device(X, shape)
    S = torch.empty(shape, dtype=torch.float64, device="cuda")
    _lib.call("b200_fss_fractions", x.data_ptr(), _device.dtype_code(x.dtype), shape[0], shape[1], shape[2], t, sub, s,
              S.data_ptr(), _device.stream_ptr())
    return S


def product_sums(S):
    """(nf, nf) float64 array: entry (i, j), i <= j, is np.sum(S[i] * S[j]) (the lower triangle is
    zero).  The fields are taken in groups of _lib.FSS_GROUP; each pair of groups is one launch."""
    nf = S.shape[0]
    P = _inputs.pixels(S.shape[1:])
    G = _lib.FSS_GROUP
    out = np.zeros((nf, nf))
    for a0 in range(0, nf, G):
        for b0 in range(a0, nf, G):
            na, nb = min(G, nf - a0), min(G, nf - b0)
            d = torch.zeros(na * nb, dtype=torch.float64, device="cuda")
            _lib.call("b200_fss_sums", S.data_ptr(), P, a0, na, b0, nb, d.data_ptr(), _device.stream_ptr())
            out[a0:a0 + na, b0:b0 + nb] += _device.to_host(d).reshape(na, nb)
    return out


def check_fields(X_f, X_o, who):
    _inputs.check(X_f, who, "X_f")
    _inputs.check(X_o, who, "X_o")
    if len(X_f.shape) != 2 or len(X_o.shape) != 2 or tuple(X_f.shape) != tuple(X_o.shape):
        raise ValueError("X_f and X_o must be two-dimensional arrays having the same shape")
    _inputs.check_pixels(_inputs.pixels(X_f.shape), who)


def fss_accum(fss, X_f, X_o):
    """Add the sums of the fractions of X_f and X_o to the accumulator."""
    who = "fss_accum"
    check_fields(X_f, X_o, who)
    s = filter_size(fss["scale"], who)
    m, n = (int(v) for v in X_f.shape)
    ff = fo = oo = np.float64(0.0)
    if m * n:
        if _inputs.np_dtype(X_f) == _inputs.np_dtype(X_o):  # one launch for both fields
            S = fractions(torch.stack([_inputs.to_device(X_f, (m, n)), _inputs.to_device(X_o, (m, n))]), (2, m, n),
                          fss["thr"], s, who)
        else:
            S = torch.cat([fractions(X, (1, m, n), fss["thr"], s, who) for X in (X_f, X_o)])
        sums = product_sums(S)
        ff, fo, oo = (np.float64(v) for v in (sums[0, 0], sums[0, 1], sums[1, 1]))
    fss["sum_obs_sq"] += oo
    fss["sum_fct_obs"] += fo
    fss["sum_fct_sq"] += ff


def fss_merge(fss_1, fss_2):
    """fss_1 with the sums of fss_2 added (a new dict)."""
    if fss_1["thr"] != fss_2["thr"]:
        raise ValueError("cannot merge: the thresholds are not same %s!=%s" % (fss_1["thr"], fss_2["thr"]))
    if fss_1["scale"] != fss_2["scale"]:
        raise ValueError("cannot merge: the scales are not same %s!=%s" % (fss_1["scale"], fss_2["scale"]))
    fss = fss_1.copy()
    for key in ("sum_obs_sq", "sum_fct_obs", "sum_fct_sq"):
        fss[key] += fss_2[key]
    return fss


def fss_compute(fss):
    """1 - MSE(S_f, S_o) / (mean S_f^2 + mean S_o^2), from the accumulated sums."""
    numer = fss["sum_fct_sq"] - 2.0 * fss["sum_fct_obs"] + fss["sum_obs_sq"]
    denom = fss["sum_fct_sq"] + fss["sum_obs_sq"]
    return 1.0 - numer / denom


def _copy_iterable(x):
    return np.copy(x) if isinstance(x, collections.abc.Iterable) else np.copy((x,))


def intensity_scale(X_f, X_o, name, thrs, scales=None, wavelet="Haar"):
    """The (scales, thresholds) table of the skill score `name` ("FSS"), scales descending, thresholds
    ascending."""
    intscale = intensity_scale_init(name, thrs, scales, wavelet)
    intensity_scale_accum(intscale, X_f, X_o)
    return intensity_scale_compute(intscale)


def intensity_scale_init(name, thrs, scales=None, wavelet="Haar"):
    """An intensity-scale accumulator: one FSS accumulator per threshold and scale."""
    kind = name.lower()
    if kind == "fss" and scales is None:
        raise ValueError("an array of spatial scales must be provided for the FSS, but %s was passed" % scales)
    if kind == "bmse" and wavelet is None:
        raise ValueError("the name of a wavelet must be provided for the BMSE, but %s was passed" % wavelet)
    if kind == "bmse":
        raise NotImplementedError("pysteps_b200 intensity_scale: the BMSE is not built on the device; use "
                                  "pysteps.verification.spatialscores.intensity_scale")
    if kind != "fss":
        raise ValueError("unknown method %s" % name)
    intscale = {"name": name, "thrs": np.sort(_copy_iterable(thrs))}
    intscale["scales"] = np.sort(_copy_iterable(scales))[::-1]
    for thr in intscale["thrs"]:
        intscale[thr] = {scale: fss_init(thr, scale) for scale in intscale["scales"]}
    intscale["label"] = "Fractions skill score"
    return intscale


def _is_fss(intscale, who):
    if intscale["name"].lower() != "fss":
        raise NotImplementedError(f"pysteps_b200 {who}: only the FSS is built on the device")


def intensity_scale_accum(intscale, X_f, X_o):
    """Accumulate X_f and X_o at every threshold and scale."""
    _is_fss(intscale, "intensity_scale_accum")
    for thr in intscale["thrs"]:
        for scale in intscale["scales"]:
            fss_accum(intscale[thr][scale], X_f, X_o)


def intensity_scale_merge(intscale_1, intscale_2):
    """intscale_1 with every FSS accumulator of intscale_2 merged in (a shallow copy)."""
    if intscale_1["name"] != intscale_2["name"]:
        raise ValueError("cannot merge: the intensity scale methods are not same %s!=%s"
                         % (intscale_1["name"], intscale_2["name"]))
    _is_fss(intscale_1, "intensity_scale_merge")
    intscale = intscale_1.copy()
    for thr in intscale["thrs"]:
        for scale in intscale["scales"]:
            intscale[thr][scale] = fss_merge(intscale[thr][scale], intscale_2[thr][scale])
    return intscale


def intensity_scale_compute(intscale):
    """The (scales, thresholds) array of FSS values."""
    _is_fss(intscale, "intensity_scale_compute")
    thrs, scales = intscale["thrs"], intscale["scales"]
    SS = np.zeros((scales.size, thrs.size))
    for i, thr in enumerate(thrs):
        for j, scale in enumerate(scales):
            SS[j, i] = fss_compute(intscale[thr][scale])
    return SS


def binary_mse(*args, **kwargs):
    """Not built on the device."""
    raise NotImplementedError("pysteps_b200 binary_mse is not built on the device; use "
                              "pysteps.verification.spatialscores.binary_mse")


def sal(*args, **kwargs):
    """Not built on the device."""
    raise NotImplementedError("pysteps_b200 sal is not built on the device; use pysteps.verification.salscores.sal")
