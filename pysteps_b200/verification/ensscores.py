"""B200 ensemble verification scores -- drop-in for ``pysteps.verification.ensscores``: ``rankhist``
and its ``rankhist_init`` / ``rankhist_accum`` / ``rankhist_compute`` steps, ``ensemble_skill`` and
``ensemble_spread``.

``ensemble_skill`` / ``ensemble_spread`` take the reference's deterministic metric names through a
table of this package (``pysteps_b200.verification.get_method`` does not dispatch them): the
categorical names run ``det_cat_fct`` per member or pair, with the reference's lower-cased score
name, so "csi" raises the reference's KeyError and "CSI" works; "fss" filters the observation and
every member once and sums every pair in batched launches (spatialscores.product_sums), bit for bit
what ``fss`` gives pair by pair; the continuous names, "binary_mse" and "sal" raise
NotImplementedError.  The mean over members or pairs is NumPy's, on the host.

``rankhist_accum`` ranks the observation among the members on the device (csrc/verification.cu):
pixels without a tie go to their bin there; for the tied pixels the uniform draws come from NumPy's
global RandomState on the host, one ``np.random.uniform(size=n_ties)`` call exactly when the
reference makes it, so that seeded workflows consume the same numbers, and reach the tied pixels in
pixel order on the device.  The accumulator is the reference's dict.  Inputs are NumPy arrays or
CUDA tensors of float32 or float64; integer dtypes, masked arrays, host tensors, 2^31 or more pixels,
more than 512 members and thresholds that are not real scalars raise NotImplementedError.
"""
import numpy as np
import torch

from .. import _device, _lib
from . import _inputs, detcatscores, detcontscores, spatialscores

# the reference's deterministic metric names (pysteps/verification/interface.py)
CATEGORICAL = ("acc", "bias", "csi", "f1", "fa", "far", "gss", "hk", "hss", "mcc", "pod", "sedi")
CONTINUOUS = ("beta", "beta1", "beta2", "corr_p", "corr_s", "drmse", "mae", "mse", "me", "nmse", "rmse", "rv",
              "scatter")


def _fss_arguments(X_f, X_o, thr, scale):
    return thr, scale


_fss_arguments.__qualname__ = "fss"  # a keyword error names the function the reference calls


def _metric(metric):
    """("fss", None) or ("call", f) with f(fct, obs, **kwargs) the per-member score of the reference's
    deterministic metric name; the names the reference does not know raise its ValueError"""
    name = "none" if metric is None else metric
    name = name.lower()
    if name in CATEGORICAL:
        def f(fct, obs, **kwargs):
            return detcatscores.det_cat_fct(fct, obs, kwargs.pop("thr"), [name])
        return "call", f
    if name in CONTINUOUS:
        def f(fct, obs, **kwargs):
            return detcontscores.det_cont_fct(fct, obs, [name], **kwargs)
        return "call", f
    if name == "fss":
        return "fss", None
    if name in ("binary_mse", "sal"):
        raise NotImplementedError(f"pysteps_b200: the deterministic score {name!r} is not built on the device; use "
                                  "pysteps.verification.ensscores")
    raise ValueError("unknown deterministic method %s" % name)


def _check_ensemble(X_f):
    if len(X_f.shape) != 3:
        raise ValueError("the number of dimensions of X_f must be equal to 3, but %i dimensions were passed"
                         % len(X_f.shape))


def _member_fractions(X_f, X_o, thr, scale, who):
    """the smoothed indicators of X_o (when given) and of every member, one tensor (k [+ 1], m, n)"""
    for name, a in (("X_f", X_f), ("X_o", X_o)):
        if a is not None:
            _inputs.check(a, who, name)
    _inputs.check_members(X_f.shape[0], who)
    k, m, n = (int(v) for v in X_f.shape)
    _inputs.check_pixels(k * m * n, who)
    s = spatialscores.filter_size(scale, who)
    parts = []
    if X_o is not None:
        parts.append(spatialscores.fractions(X_o, (1, m, n), thr, s, who))
    parts.append(spatialscores.fractions(X_f, (k, m, n), thr, s, who))
    return torch.cat(parts) if len(parts) > 1 else parts[0]


def _fss_of(oo, fo, ff):
    d = spatialscores.fss_init(None, None)
    d["sum_obs_sq"] += np.float64(oo)
    d["sum_fct_obs"] += np.float64(fo)
    d["sum_fct_sq"] += np.float64(ff)
    return spatialscores.fss_compute(d)


def ensemble_skill(X_f, X_o, metric, **kwargs):
    """The mean over the k members of X_f (k, m, n) of the deterministic score `metric` against X_o."""
    _check_ensemble(X_f)
    if tuple(X_f.shape[1:]) != tuple(X_o.shape):
        raise ValueError("the shape of X_f does not match the shape of X_o (%d,%d)!=(%d,%d)"
                         % (X_f.shape[1], X_f.shape[2], X_o.shape[0], X_o.shape[1]))
    kind, f = _metric(metric)
    k = X_f.shape[0]
    skill = []
    if kind == "fss" and k > 0:
        thr, scale = _fss_arguments(X_f, X_o, **kwargs)
        sums = spatialscores.product_sums(_member_fractions(X_f, X_o, thr, scale, "ensemble_skill"))
        for i in range(1, k + 1):
            skill.append(_fss_of(sums[0, 0], sums[0, i], sums[i, i]))
        return np.mean(skill)
    for member in range(k):
        s = f(X_f[member, :, :], X_o, **kwargs)
        skill.append(s[metric] if isinstance(s, dict) else s)
    return np.mean(skill)


def ensemble_spread(X_f, metric, **kwargs):
    """The mean over the k (k - 1) / 2 member pairs of X_f (k, m, n) of the deterministic score `metric`
    of one member against the other."""
    _check_ensemble(X_f)
    k = X_f.shape[0]
    if k < 2:
        raise ValueError("the number of members in X_f must be greater than 1, but %i members were passed" % k)
    kind, f = _metric(metric)
    spread = []
    if kind == "fss":
        thr, scale = _fss_arguments(X_f, X_f, **kwargs)
        sums = spatialscores.product_sums(_member_fractions(X_f, None, thr, scale, "ensemble_spread"))
        for i in range(k):
            for j in range(i + 1, k):
                spread.append(_fss_of(sums[j, j], sums[i, j], sums[i, i]))
        return np.mean(spread)
    for i in range(k):
        for j in range(i + 1, k):
            s = f(X_f[i, :, :], X_f[j, :, :], **kwargs)
            spread.append(s[metric] if isinstance(s, dict) else s)
    return np.mean(spread)


def rankhist(X_f, X_o, X_min=None, normalize=True):
    """The rank histogram of the observations X_o (m, n, ...) among the k members of X_f (k, m, n,
    ...), normalised to sum to one when normalize is true; with X_min, the pixels where the members
    and the observation are all below X_min are left out."""
    rhist = rankhist_init(X_f.shape[0], X_min)
    rankhist_accum(rhist, X_f, X_o)
    return rankhist_compute(rhist, normalize)


def rankhist_init(num_ens_members, X_min=None):
    """A rank-histogram accumulator of num_ens_members + 1 bins."""
    return dict(num_ens_members=num_ens_members, n=np.zeros(num_ens_members + 1, dtype=int), X_min=X_min)


def rankhist_accum(rankhist, X_f, X_o):
    """Add the ranks of X_o among the members of X_f to the accumulator."""
    who = "rankhist_accum"
    k_dict = rankhist["num_ens_members"]
    if X_f.shape[0] != k_dict:
        raise ValueError(
            "the number of ensemble members in X_f does not match the number of members in the rank "
            "histogram (%d!=%d)" % (X_f.shape[0], k_dict)
        )
    _inputs.check(X_f, who, "X_f")
    _inputs.check(X_o, who, "X_o")
    shapes = _inputs.ensemble_shapes(tuple(X_f.shape), tuple(X_o.shape), obs_first=True)
    if not shapes:
        raise NotImplementedError(f"pysteps_b200 {who}: shapes {tuple(X_f.shape)} and {tuple(X_o.shape)}")
    if shapes == "empty":
        X_f, X_o = _inputs.empty(X_f, (X_f.shape[0], 0)), _inputs.empty(X_o, (0,))
    k, N = int(X_f.shape[0]), _inputs.pixels(X_f.shape[1:])
    _inputs.check_members(k, who)
    _inputs.check_pixels(N, who)
    X_min = rankhist["X_min"]
    fdt, odt = _inputs.np_dtype(X_f), _inputs.np_dtype(X_o)
    if X_min is None:
        use_min, thr_f, sub_f, thr_o, sub_o = 0, 0.0, 0.0, 0.0, 0.0
    else:
        use_min = 1
        thr_f = _inputs.threshold(fdt, X_min, who)
        thr_o = _inputs.threshold(odt, X_min, who)
        below = X_min - 1  # stored into each array, so rounded to its dtype
        sub_f, sub_o = float(np.asarray(below).astype(fdt)), float(np.asarray(below).astype(odt))
    f = _inputs.to_device(X_f, (k, N))
    o = _inputs.to_device(X_o, (N,))
    hist = torch.empty(k + 1, dtype=torch.int64, device="cuda")
    ties = torch.empty((max(N, 1), 2), dtype=torch.int32, device="cuda")
    d_ties = torch.empty(1, dtype=torch.int64, device="cuda")
    stream = _device.stream_ptr()
    _lib.call("b200_verif_rankhist", f.data_ptr(), _device.dtype_code(f.dtype), o.data_ptr(),
              _device.dtype_code(o.dtype), k, N, use_min, thr_f, sub_f, thr_o, sub_o, hist.data_ptr(),
              ties.data_ptr(), d_ties.data_ptr(), stream)
    n_ties = int(_device.to_host(d_ties)[0])
    if n_ties > 0:
        u = np.random.uniform(low=0.0, high=1.0, size=n_ties)
        d_u = _device.to_device(u)
        _lib.call("b200_verif_rankhist_ties", ties.data_ptr(), n_ties, _device.ptr(d_u), k, hist.data_ptr(), stream)
    rankhist["n"] += _device.to_host(hist)


def rankhist_compute(rankhist, normalize=True):
    """The k + 1 bin counts, or their fractions of the total when normalize is true."""
    counts = rankhist["n"]
    if not normalize:
        return counts
    return counts * 1.0 / sum(counts)
