"""B200 ensemble statistics -- drop-ins for ``mean``, ``excprob`` and ``banddepth`` of
``pysteps.postprocessing.ensemblestats`` (pysteps/postprocessing/ensemblestats.py:20-179).

Reductions over the member axis, on the device (csrc/ensemblestats.cu):
  * ``mean``: the sequential sum over members in X's dtype, divided by k -- what NumPy computes when
    the member axis is outermost in memory (C order, and views such as ``R_f[:, -1]``); the nanmean
    form (``ignore_nan`` or ``X_thr``) divides float64(sum) by the integer count of members.  When
    the member axis is not outermost (Fortran order), NumPy sums pairwise and the results differ by
    rounding only (DESIGN.md section 4).
  * ``excprob``: exact counts of the members >= every threshold, in one pass for up to 8 thresholds.
  * ``banddepth``: the mask and its column scan on the device; the tie-breaks ``np.random.random((k,
    p))`` are drawn on the host from NumPy's global RandomState, as the reference draws them, so that
    seeded workflows consume the same numbers; the member ranks and their int64 sums on the device;
    the reference's own float64 tail on the host.

Signatures, exceptions and warnings are the reference's; a warning that depends on pixel values
comes from a flag the kernel sets.  Thresholds are compared in NumPy's result dtype (NEP 50,
``pysteps_b200/_compare.py``).  NumPy input returns NumPy; a CUDA-tensor X returns a CUDA tensor.
Only float32 and float64 ensembles are supported; integer dtypes, masked arrays, frames of 2^31
pixels or more and other thresholds raise NotImplementedError (there is no CPU path).

Parity: tests/test_ensemblestats_gpu.py (device), tests/test_oracle_ensemblestats.py and
tests/test_host_logic_ensemblestats.py (oracle and host logic on the CPU).
"""
import warnings

import numpy as np
import torch
from scipy.special import comb

from .. import _compare, _device, _lib

_OVERFLOW, _INVALID, _EMPTY = 1, 2, 4  # B200_ENSEMBLE_OVERFLOW / _INVALID / _EMPTY


def mean(X, ignore_nan=False, X_thr=None):
    """Same contract as the reference: X (k, m, n) or (m, n); returns the (m, n) mean in X's dtype.
    ignore_nan: skip NaN members; X_thr: skip the members below it."""
    X = _as_array(X, "mean")
    X_ndim = X.ndim

    if X_ndim > 3 or X_ndim <= 1:
        raise Exception(
            "Number of dimensions of X should be 2 or 3." + "It was: {}".format(X_ndim)
        )
    elif X.ndim == 2:
        X = X[None, ...]

    _check_supported(X, "mean")
    nan_mode = bool(ignore_nan or X_thr is not None)
    use_thr = X_thr is not None
    thr = _threshold(X, X_thr, "mean") if use_thr else 0.0
    k, N, d = _members(X)
    out = torch.empty(X.shape[1:], dtype=d.dtype, device="cuda")
    flags = torch.empty(1, dtype=torch.int32, device="cuda")
    _lib.call("b200_ensemble_mean", d.data_ptr(), _device.dtype_code(d.dtype), k, N, int(nan_mode), int(use_thr),
              thr, out.data_ptr(), flags.data_ptr(), _device.stream_ptr())
    fl = int(_device.to_host(flags)[0])
    if nan_mode:
        # np.nanmean: the sum, then the division (its warnings suppressed), then the empty slices
        _reduce_warnings(fl)
        if fl & _EMPTY:
            warnings.warn("Mean of empty slice", RuntimeWarning, stacklevel=2)
    else:
        # np.mean: the empty axis, the sum, then the division by k
        if k == 0:
            warnings.warn("Mean of empty slice.", RuntimeWarning, stacklevel=2)
        _reduce_warnings(fl)
        if k == 0 and N > 0:
            _fp_error("invalid", "invalid value encountered in divide")
    return _result(out, X)


def excprob(X, X_thr, ignore_nan=False):
    """Same contract as the reference: X (k, m, n, ...); X_thr a threshold or a sequence of them;
    returns the float64 exceedance probabilities (len(X_thr), m, n, ...), without the first axis for
    a scalar threshold."""
    X = _as_array(X, "excprob")
    X_ndim = X.ndim

    if X_ndim < 3:
        raise Exception(
            f"Number of dimensions of X should be 3 or more. It was: {X_ndim}"
        )

    if np.isscalar(X_thr):
        X_thr = [X_thr]
        scalar_thr = True
    else:
        scalar_thr = False
    thresholds = [x for x in X_thr]  # a 0-d array raises TypeError here, as in the reference's loop
    if not thresholds and not scalar_thr:
        np.stack([])  # the reference's ValueError: need at least one array to stack

    _check_supported(X, "excprob")
    thr = np.array([_threshold(X, x, "excprob") for x in thresholds], dtype=np.float64)
    k, N, d = _members(X)
    out = torch.empty((len(thr),) + tuple(X.shape[1:]), dtype=torch.float64, device="cuda")
    flags = torch.empty(1, dtype=torch.int32, device="cuda")
    _lib.call("b200_ensemble_excprob", d.data_ptr(), _device.dtype_code(d.dtype), k, N,
              thr.ctypes.data_as(_lib.c_dp), len(thr), int(bool(ignore_nan)), out.data_ptr(), flags.data_ptr(),
              _device.stream_ptr())
    fl = int(_device.to_host(flags)[0])
    for _ in thresholds:  # the reference averages once per threshold
        if ignore_nan:
            if fl & _EMPTY:
                warnings.warn("Mean of empty slice", RuntimeWarning, stacklevel=2)
        elif k == 0:
            warnings.warn("Mean of empty slice.", RuntimeWarning, stacklevel=2)
            if N > 0:
                _fp_error("invalid", "invalid value encountered in divide")
    return _result(out[0] if scalar_thr else out, X)


def banddepth(X, thr=None, norm=False):
    """Same contract as the reference: X (k, m, ...); returns the float64 modified band depth of
    every member, shape (k,), normalised to [0, 1] with norm=True.  The random tie-breaks come from
    NumPy's global RandomState, exactly as in the reference."""
    if not (isinstance(X, np.ndarray) or _device.is_device_tensor(X)):
        raise NotImplementedError("pysteps_b200 banddepth: X must be a NumPy array or a CUDA tensor")
    _check_supported(X, "banddepth")
    if X.ndim < 2:
        raise NotImplementedError("pysteps_b200 banddepth: X must have a member axis and a pixel axis")
    k, N, d = _members(X)
    code = _device.dtype_code(d.dtype)
    np_dtype = np.float32 if d.dtype == torch.float32 else np.float64

    # mask invalid pixels
    if thr is None:
        if d.numel() == 0:
            raise ValueError("zero-size array to reduction operation fmin which has no identity")
        stats = torch.empty(4, dtype=torch.float64, device="cuda")
        _lib.call("b200_field_stats", d.data_ptr(), code, d.numel(), stats.data_ptr(), _device.stream_ptr())
        nanmin, n_nan = (float(v) for v in _device.to_host(stats)[[1, 3]])
        if n_nan == d.numel():
            warnings.warn("All-NaN slice encountered", RuntimeWarning, stacklevel=2)
        thr = np_dtype(nanmin)  # np.nanmin returns a scalar of X's dtype
    t = _threshold(np.zeros(1, np_dtype), thr, "banddepth")
    col = torch.empty(max(N, 1), dtype=torch.int32, device="cuda")
    d_p = torch.empty(1, dtype=torch.int64, device="cuda")
    _lib.call("b200_ensemble_band_mask", d.data_ptr(), code, k, N, t, col.data_ptr(), d_p.data_ptr(),
              _device.stream_ptr())

    n = X.shape[0]
    p = np.int64(_device.to_host(d_p)[0])  # np.sum(mask)

    # assign ranks
    b = np.random.random((n, p))
    d_b = _device.to_device(b)
    match = torch.empty(max(k, 1), dtype=torch.int64, device="cuda")
    _lib.call("b200_ensemble_band_match", d.data_ptr(), code, k, N, col.data_ptr(), _device.ptr(d_b) if p else None,
              int(p), match.data_ptr(), _device.stream_ptr())
    match = _device.to_host(match)[:k]  # np.sum(match, axis=1): int64

    # compute band depth
    nchoose2 = comb(n, 2)
    proportion = match / p
    depth = (proportion + n - 1) / nchoose2

    # normalize depth between 0 and 1
    if norm:
        depth = (depth - depth.min()) / (depth.max() - depth.min())

    return torch.from_numpy(depth).to("cuda") if _device.is_device_tensor(X) else depth


def _as_array(X, who):
    """np.asanyarray(X) as the reference does, a CUDA tensor as it is; masked arrays and host tensors
    are not supported"""
    if _device.is_device_tensor(X):
        return X
    if isinstance(X, torch.Tensor):
        raise NotImplementedError(f"pysteps_b200 {who}: X must be a NumPy array or a CUDA tensor")
    return np.asanyarray(X)


def _check_supported(X, who):
    if isinstance(X, np.ma.MaskedArray):
        raise NotImplementedError(f"pysteps_b200 {who}: masked arrays are not supported")
    lib = torch if isinstance(X, torch.Tensor) else np
    if X.dtype not in (lib.float32, lib.float64):
        raise NotImplementedError(f"pysteps_b200 {who}: ensembles of dtype {X.dtype} are not supported "
                                  "(float32 or float64)")
    if int(np.prod(X.shape[1:], dtype=np.int64)) >= 1 << 31:
        raise NotImplementedError(f"pysteps_b200 {who}: 2^31 pixels or more per member are not supported")


def _threshold(X, thr, who):
    """thr as the float64 the kernels compare with (rounded to NumPy's comparison dtype)"""
    if isinstance(thr, np.ndarray) and thr.ndim > 0 or isinstance(thr, (list, tuple, torch.Tensor)):
        raise NotImplementedError(f"pysteps_b200 {who}: thresholds must be scalars")
    dt = np.float32 if X.dtype in (np.float32, torch.float32) else np.float64
    return _compare.comparison_threshold(dt, thr, who)[0]


def _members(X):
    """(k, N, d): the member count, the pixels per member and the ensemble as a C-contiguous (k, N)
    device tensor of X's dtype"""
    k = int(X.shape[0])
    N = int(np.prod(X.shape[1:], dtype=np.int64))
    _device.require_cuda()
    d = X.contiguous() if isinstance(X, torch.Tensor) else _device.to_device(np.asarray(X))
    return k, N, d.reshape(k, N)


def _result(out, X):
    return out if _device.is_device_tensor(X) else _device.to_host(out)


def _fp_error(kind, message):
    """A floating-point error as NumPy reports it under the current np.errstate"""
    mode = np.geterr()[kind]
    if mode == "ignore":
        return
    if mode == "raise":
        raise FloatingPointError(message)
    warnings.warn(message, RuntimeWarning, stacklevel=3)


def _reduce_warnings(fl):
    """the errors of NumPy's sum over the members, in NumPy's order"""
    if fl & _OVERFLOW:
        _fp_error("over", "overflow encountered in reduce")
    if fl & _INVALID:
        _fp_error("invalid", "invalid value encountered in reduce")
