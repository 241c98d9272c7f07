"""B200 probabilistic verification scores -- drop-ins for ``CRPS``, ``reldiag`` and ``ROC_curve`` of
``pysteps.verification.probscores`` and their ``*_init`` / ``*_accum`` / ``*_compute`` steps.

Only ``*_accum`` touches the device (csrc/verification.cu); ``*_init`` and ``*_compute`` are the few
lines of host arithmetic of the reference.  The accumulator objects are the reference's dicts, with
its keys and value types, so a dict made by pysteps can be accumulated here and finished by pysteps,
and the reverse.
  * ``CRPS_accum``: per pixel the k members sorted, the k + 1 alpha / beta terms in the reference's
    dtypes, NumPy's pairwise sum over them, and NumPy's pairwise sum of those over the pixels.
  * ``reldiag_accum``: np.digitize over the float64 bin edges of the dict, the exact per-bin counts,
    and NumPy's pairwise sum of the probabilities of every bin in pixel order and in their dtype.
  * ``ROC_curve_accum``: the exact hits, misses, false alarms and correct negatives of every
    threshold from one pass.
Inputs are NumPy arrays or CUDA tensors of float32 or float64 in any combination; the results are
the reference's host scalars and arrays either way.  Integer dtypes, masked arrays, host tensors,
2^31 or more pixels, more than 512 members, more than 2048 bins or thresholds, unsorted bin edges
or thresholds and thresholds that are not real scalars raise NotImplementedError: there is no CPU
path.
"""
import numpy as np
import torch

from .. import _device, _lib
from . import _inputs


def CRPS(X_f, X_o):
    """The continuous ranked probability score of the ensemble X_f (k, m, n, ...) against the
    observations X_o (m, n, ...), averaged over the pixels where all are finite."""
    crps = CRPS_init()
    CRPS_accum(crps, X_f, X_o)
    return CRPS_compute(crps)


def CRPS_init():
    """A CRPS accumulator: the running sum of the per-pixel scores and their number."""
    return dict(CRPS_sum=0.0, n=0.0)


def CRPS_accum(CRPS, X_f, X_o):
    """Add the per-pixel CRPS of X_f (k, m, n, ...) against X_o (m, n, ...) to the accumulator."""
    who = "CRPS_accum"
    _inputs.check(X_f, who, "X_f")
    _inputs.check(X_o, who, "X_o")
    shapes = _inputs.ensemble_shapes(tuple(X_f.shape), tuple(X_o.shape))
    if not shapes:
        raise NotImplementedError(f"pysteps_b200 {who}: shapes {tuple(X_f.shape)} and {tuple(X_o.shape)}")
    if shapes == "empty":
        X_f, X_o = _inputs.empty(X_f, (X_f.shape[0], 0)), _inputs.empty(X_o, (0,))
    k, N = int(X_f.shape[0]), _inputs.pixels(X_f.shape[1:])
    _inputs.check_members(k, who)
    _inputs.check_pixels(N, who)
    f = _inputs.to_device(X_f, (k, N))
    o = _inputs.to_device(X_o, (N,))
    res = torch.empty(max(N, 1), dtype=torch.float64, device="cuda")
    d_n = torch.empty(1, dtype=torch.int64, device="cuda")
    stream = _device.stream_ptr()
    _lib.call("b200_verif_crps", f.data_ptr(), _device.dtype_code(f.dtype), o.data_ptr(), _device.dtype_code(o.dtype),
              k, N, res.data_ptr(), d_n.data_ptr(), stream)
    n = int(_device.to_host(d_n)[0])
    total = torch.empty(1, dtype=torch.float64, device="cuda")
    off, count = np.zeros(1, np.int64), np.array([n], np.int64)  # host segment table, alive for the call
    _lib.call("b200_pairwise_sum", res.data_ptr(), _lib.F64, off.ctypes.data, count.ctypes.data, 1,
              total.data_ptr(), stream)
    CRPS["CRPS_sum"] += _device.to_host(total)[0]  # np.float64, as np.sum returns
    CRPS["n"] += n


def CRPS_compute(CRPS):
    """The mean CRPS of the accumulator."""
    total = 1.0 * CRPS["CRPS_sum"]
    return total / CRPS["n"]


def reldiag(P_f, X_o, X_min, n_bins=10, min_count=10):
    """The x- and y-coordinates of the reliability diagram of the probabilities P_f of exceeding
    X_min against the observations X_o."""
    rdiag = reldiag_init(X_min, n_bins, min_count)
    reldiag_accum(rdiag, P_f, X_o)
    return reldiag_compute(rdiag)


def reldiag_init(X_min, n_bins=10, min_count=10):
    """A reliability-diagram accumulator of n_bins bins; bins with fewer than min_count pairs in
    one accumulation add nothing."""
    edges = np.linspace(-1e-6, 1 + 1e-6, int(n_bins + 1))
    out = dict(X_min=X_min, bin_edges=edges, n_bins=n_bins)
    out["X_sum"] = np.zeros(n_bins)
    for key in ("Y_sum", "num_idx", "sample_size"):
        out[key] = np.zeros(n_bins, dtype=int)
    out["min_count"] = min_count
    return out


def reldiag_accum(reldiag, P_f, X_o):
    """Add the probability-observation pairs where both are finite to the accumulator."""
    who = "reldiag_accum"
    _inputs.check(P_f, who, "P_f")
    _inputs.check(X_o, who, "X_o")
    shapes = _inputs.pair_shapes(tuple(P_f.shape), tuple(X_o.shape))
    if not shapes:
        raise NotImplementedError(f"pysteps_b200 {who}: shapes {tuple(P_f.shape)} and {tuple(X_o.shape)}")
    if shapes == "empty":
        P_f, X_o = _inputs.empty(P_f, (0,)), _inputs.empty(X_o, (0,))
    N = _inputs.pixels(P_f.shape)
    _inputs.check_pixels(N, who)
    edges = np.ascontiguousarray(reldiag["bin_edges"], dtype=np.float64)
    nb = len(edges) - 1
    if edges.ndim != 1 or nb < 0 or nb > _lib.VERIF_MAX_BINS or np.any(edges[1:] < edges[:-1]) \
            or not np.all(np.isfinite(edges)):
        raise NotImplementedError(f"pysteps_b200 {who}: up to {_lib.VERIF_MAX_BINS} bins with finite increasing "
                                  "edges are supported")
    thr = _inputs.threshold(_inputs.np_dtype(X_o), reldiag["X_min"], who)
    p = _inputs.to_device(P_f, (N,))
    o = _inputs.to_device(X_o, (N,))
    sorted_p = torch.empty(max(N, 1), dtype=p.dtype, device="cuda")
    seg = torch.empty(nb + 1, dtype=torch.int64, device="cuda")
    above = torch.empty(max(nb, 1), dtype=torch.int64, device="cuda")
    stream = _device.stream_ptr()
    code = _device.dtype_code(p.dtype)
    _lib.call("b200_verif_reldiag", p.data_ptr(), code, o.data_ptr(), _device.dtype_code(o.dtype), N,
              edges.ctypes.data_as(_lib.c_dp), nb + 1, thr, sorted_p.data_ptr(), seg.data_ptr(), above.data_ptr(),
              stream)
    start = _device.to_host(seg)
    count = np.diff(start)
    sums = torch.empty(max(nb, 1), dtype=p.dtype, device="cuda")
    if nb:
        off = np.ascontiguousarray(start[:-1])
        _lib.call("b200_pairwise_sum", sorted_p.data_ptr(), code, off.ctypes.data, count.ctypes.data, nb,
                  sums.data_ptr(), stream)
    sums = _device.to_host(sums)[:nb]
    above = _device.to_host(above)[:nb]

    keep = np.array([int(c) >= reldiag["min_count"] for c in count], dtype=bool)
    x = np.where(keep, sums.astype(np.float64), 0.0)
    reldiag["X_sum"] += x
    reldiag["Y_sum"] += np.where(keep, above, 0)
    reldiag["num_idx"] += np.where(keep, count, 0)
    reldiag["sample_size"] += [int(c) if kept else 0 for c, kept in zip(count, keep)]  # a list, as NumPy types it


def reldiag_compute(reldiag):
    """The x- and y-coordinates (mean probability, observed frequency) of every bin."""
    n = reldiag["num_idx"]
    y = 1.0 * reldiag["Y_sum"] / n
    x = 1.0 * reldiag["X_sum"] / n
    return x, y


def ROC_curve(P_f, X_o, X_min, n_prob_thrs=10, compute_area=False):
    """The probability of false detection and of detection at n_prob_thrs probability thresholds
    evenly spaced in [0, 1], and with compute_area the area under the curve."""
    roc = ROC_curve_init(X_min, n_prob_thrs)
    ROC_curve_accum(roc, P_f, X_o)
    return ROC_curve_compute(roc, compute_area)


def ROC_curve_init(X_min, n_prob_thrs=10):
    """A ROC accumulator: the four contingency counts at every probability threshold."""
    out = dict(X_min=X_min)
    for key in ("hits", "misses", "false_alarms", "corr_neg"):
        out[key] = np.zeros(n_prob_thrs, dtype=int)
    out["prob_thrs"] = np.linspace(0.0, 1.0, int(n_prob_thrs))
    return out


def ROC_curve_accum(ROC, P_f, X_o):
    """Add the probability-observation pairs where both are finite to the accumulator."""
    who = "ROC_curve_accum"
    _inputs.check(P_f, who, "P_f")
    _inputs.check(X_o, who, "X_o")
    shapes = _inputs.pair_shapes(tuple(P_f.shape), tuple(X_o.shape))
    if not shapes:
        raise NotImplementedError(f"pysteps_b200 {who}: shapes {tuple(P_f.shape)} and {tuple(X_o.shape)}")
    if shapes == "empty":
        P_f, X_o = _inputs.empty(P_f, (0,)), _inputs.empty(X_o, (0,))
    N = _inputs.pixels(P_f.shape)
    _inputs.check_pixels(N, who)
    thrs = np.ascontiguousarray(ROC["prob_thrs"], dtype=np.float64)
    T = len(thrs)
    if thrs.ndim != 1 or T > _lib.VERIF_MAX_BINS or np.any(thrs[1:] < thrs[:-1]) or np.any(np.isnan(thrs)):
        raise NotImplementedError(f"pysteps_b200 {who}: up to {_lib.VERIF_MAX_BINS} increasing thresholds are "
                                  "supported")
    thr = _inputs.threshold(_inputs.np_dtype(X_o), ROC["X_min"], who)
    p = _inputs.to_device(P_f, (N,))
    o = _inputs.to_device(X_o, (N,))
    counts = torch.empty(2 * (T + 1), dtype=torch.int64, device="cuda")
    _lib.call("b200_verif_roc", p.data_ptr(), _device.dtype_code(p.dtype), o.data_ptr(), _device.dtype_code(o.dtype),
              N, thrs.ctypes.data_as(_lib.c_dp), T, thr, counts.data_ptr(), _device.stream_ptr())
    counts = _device.to_host(counts)
    # pairs with c thresholds <= P: P >= thrs[i] exactly for i < c
    event, other = counts[:T + 1], counts[T + 1:]
    hits = np.cumsum(event[::-1])[::-1][1:]
    false_alarms = np.cumsum(other[::-1])[::-1][1:]
    ROC["hits"] += hits
    ROC["misses"] += event.sum() - hits
    ROC["false_alarms"] += false_alarms
    ROC["corr_neg"] += other.sum() - false_alarms


def ROC_curve_compute(ROC, compute_area=False):
    """The lists of POFD and POD at every threshold, and with compute_area the area under the curve
    (trapezoids between the points, closed at (1, 1) and (0, 0))."""
    pod, pofd = [], []
    for i in range(len(ROC["prob_thrs"])):
        h, m = ROC["hits"][i], ROC["misses"][i]
        fa, cn = ROC["false_alarms"][i], ROC["corr_neg"][i]
        pod.append(1.0 * h / (h + m))
        pofd.append(1.0 * fa / (cn + fa))
    if not compute_area:
        return pofd, pod
    area = (1.0 - pofd[0]) * (1.0 + pod[0]) / 2.0
    for i in range(len(pod) - 1):
        area += (pofd[i] - pofd[i + 1]) * (pod[i + 1] + pod[i]) / 2.0
    area += pofd[-1] * pod[-1] / 2.0
    return pofd, pod, area
