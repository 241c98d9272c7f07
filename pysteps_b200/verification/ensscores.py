"""B200 ensemble verification score -- drop-in for ``rankhist`` of ``pysteps.verification.ensscores``
and its ``rankhist_init`` / ``rankhist_accum`` / ``rankhist_compute`` steps.

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
from . import _inputs


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
