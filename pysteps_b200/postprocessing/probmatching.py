"""B200 probability matching -- drop-ins for ``nonparam_match_empirical_cdf`` and
``resample_distributions`` of ``pysteps.postprocessing.probmatching``
(pysteps/postprocessing/probmatching.py:55-140, 277-337).

Both sort on the device (csrc/probmatching.cu, on the radix sort of csrc/radix_sort.cuh):
  * ``nonparam_match_empirical_cdf``: one call gathers the minima and counts the host needs for the
    reference's errors, its warning and its percentile branch, and reads them back.  The host computes
    the order-statistic indices and ``gamma`` of ``np.percentile`` with NumPy's own expressions; the
    device interpolates.  Only the values above each array's minimum are sorted, so the cost follows the
    rain area.
  * ``resample_distributions``: the NaN count is read back (it decides the output dtype); the 0/1 draws
    come from ``randgen.binomial(1, p, n)`` on the host, exactly as the reference draws them, so that
    seeded workflows consume the same stream.

Ties.  NumPy's default ``argsort`` is not stable, and its tie order depends on the CPU it runs on.  The
device ranks equal initial values in pixel order, as ``argsort(kind="stable")`` does.  The output is
bit-identical to the reference wherever the initial array's values above its minimum are distinct;
otherwise it is bit-identical to the reference with a stable argsort, and holds the same multiset of
values within every group of tied pixels.  The same holds for -0.0 against +0.0 among tied values: a
dry target value is written as the target's minimum, -0.0 when some minimal value is -0.0.

Signatures, exceptions and warnings are the reference's.  NumPy input returns NumPy; a CUDA-tensor
input returns a CUDA tensor, and every launch runs on the calling thread's current stream.  Only
float32 and float64 arrays are supported; integer dtypes, masked arrays and arrays of 2^31 values or
more raise NotImplementedError before any launch (there is no CPU path).

Parity: tests/test_probmatching_gpu.py (device), tests/test_oracle_probmatching.py and
tests/test_host_logic_probmatching.py (oracle and host logic on the CPU).
"""
import ctypes
import warnings

import numpy as np
import torch

from .. import _device, _lib


def nonparam_match_empirical_cdf(initial_array, target_array, ignore_indices=None):
    """Same contract as the reference: the float64 array of initial_array's shape whose values are
    target_array's, assigned in the rank order of initial_array; the pixels at initial_array's
    minimum get target_array's minimum and the pixels at ignore_indices (an index or a boolean mask)
    keep initial_array's values."""
    for a in (initial_array, target_array):
        _check_supported(a, "nonparam_match_empirical_cdf")
    _device.require_cuda()
    x, t = _flat(initial_array), _flat(target_array)
    n, n_t = x.numel(), t.numel()
    mask, mask_error = None, None
    if ignore_indices is not None:
        try:
            mask = _ignore_mask(ignore_indices, tuple(initial_array.shape), n)
        except (IndexError, TypeError, ValueError) as e:  # raised where the reference indexes, after its checks
            mask_error = e

    scratch = _scratch(max(n, n_t))
    stats = torch.empty(8, dtype=torch.float64, device="cuda")
    _lib.call("b200_pm_match_stats", x.data_ptr(), _device.dtype_code(x.dtype), _device.ptr(mask), n, t.data_ptr(),
              _device.dtype_code(t.dtype), n_t, stats.data_ptr(), scratch.data_ptr(), scratch.numel(),
              _device.stream_ptr())
    zvalue, x_notnan, x_nonfinite, x_masked, x_wet, _, t_notnan, t_wet = _device.to_host(stats).tolist()

    if x_notnan == 0:
        raise ValueError("Initial array contains only nans.")
    if n != n_t:
        raise ValueError(
            "dimension mismatch between initial_array and target_array: "
            f"initial_array.shape={_shape(initial_array)}, target_array.shape={_shape(target_array)}"
        )
    if mask_error is not None:
        raise mask_error
    # the masked pixels take the value zvalue, which is not finite when the minimum is -inf or +inf
    if x_nonfinite or (x_masked and not np.isfinite(zvalue)):
        raise ValueError(
            "Initial array contains non-finite values outside ignore_indices mask."
        )
    if t_notnan == 0:
        warnings.warn("All-NaN slice encountered", RuntimeWarning, stacklevel=2)

    x_wet, t_wet = int(x_wet), int(t_wet)
    clip = t_wet > x_wet
    i0, i1, gamma = _percentile_taps(n, x_wet) if clip else (0, 0, 0.0)
    out = torch.empty(tuple(initial_array.shape), dtype=torch.float64, device="cuda")
    _lib.call("b200_pm_match", x.data_ptr(), _device.dtype_code(x.dtype), _device.ptr(mask), t.data_ptr(),
              _device.dtype_code(t.dtype), n, stats.data_ptr(), x_wet, t_wet, int(clip), i0, i1, gamma,
              out.data_ptr(), scratch.data_ptr(), scratch.numel(), _device.stream_ptr())
    return out if _device.is_device_tensor(initial_array) else _device.to_host(out)


def resample_distributions(first_array, second_array, probability_first_array, randgen=np.random):
    """Same contract as the reference: the values of the two arrays that are NaN in neither, each
    sorted in descending order, picked from first_array with probability probability_first_array
    (clipped to [0, 1]) by randgen.binomial, sorted again in descending order behind the NaNs; a 1-D
    array of the arrays' size."""
    if first_array.shape != second_array.shape:
        raise ValueError("first_array and second_array must have the same shape")
    for a in (first_array, second_array):
        _check_supported(a, "resample_distributions")
    probability_first_array = np.clip(probability_first_array, 0.0, 1.0)
    _device.require_cuda()
    a, b = _flat(first_array), _flat(second_array)
    n = a.numel()
    n_nan = torch.empty(1, dtype=torch.int64, device="cuda")
    _lib.call("b200_pm_resample_nan", a.data_ptr(), _device.dtype_code(a.dtype), b.data_ptr(),
              _device.dtype_code(b.dtype), n, n_nan.data_ptr(), _device.stream_ptr())
    n_nan = int(_device.to_host(n_nan)[0])
    # the NaNs make both arrays float64; otherwise np.where's result type
    dtype = torch.float64 if n_nan or torch.float64 in (a.dtype, b.dtype) else torch.float32

    draws = randgen.binomial(1, probability_first_array, n).astype(bool)
    out = torch.empty(n, dtype=dtype, device="cuda")
    if n:
        d_draws = _device.to_device(draws.view(np.uint8))
        scratch = _scratch(n)
        _lib.call("b200_pm_resample", a.data_ptr(), _device.dtype_code(a.dtype), b.data_ptr(),
                  _device.dtype_code(b.dtype), n, n_nan, d_draws.data_ptr(), out.data_ptr(),
                  _device.dtype_code(dtype), scratch.data_ptr(), scratch.numel(), _device.stream_ptr())
    on_device = _device.is_device_tensor(first_array) or _device.is_device_tensor(second_array)
    return out if on_device else _device.to_host(out)


def _check_supported(a, who):
    if not (isinstance(a, np.ndarray) or _device.is_device_tensor(a)):
        raise NotImplementedError(f"pysteps_b200 {who}: arrays must be NumPy arrays or CUDA tensors")
    if isinstance(a, np.ma.MaskedArray):
        raise NotImplementedError(f"pysteps_b200 {who}: masked arrays are not supported")
    lib = torch if isinstance(a, torch.Tensor) else np
    if a.dtype not in (lib.float32, lib.float64):
        raise NotImplementedError(f"pysteps_b200 {who}: arrays of dtype {a.dtype} are not supported "
                                  "(float32 or float64)")
    if int(np.prod(a.shape, dtype=np.int64)) >= 1 << 31:
        raise NotImplementedError(f"pysteps_b200 {who}: arrays of 2^31 values or more are not supported")


def _flat(a):
    """a as a flat C-contiguous device tensor of its dtype"""
    d = a.contiguous() if isinstance(a, torch.Tensor) else _device.to_device(np.asarray(a))
    return d.reshape(-1)


def _shape(a):
    return tuple(a.shape)


def _ignore_mask(ignore_indices, shape, n):
    """ignore_indices as a flat device mask of n bytes: a CUDA bool tensor of n values as it is, any
    NumPy index through a boolean array of the initial array's shape (the reference's two assignments
    at that index touch exactly the pixels of that mask)"""
    if isinstance(ignore_indices, torch.Tensor):
        if not (ignore_indices.is_cuda and ignore_indices.dtype == torch.bool and ignore_indices.numel() == n):
            raise NotImplementedError("pysteps_b200 nonparam_match_empirical_cdf: a tensor ignore_indices must be a "
                                      "CUDA bool tensor of the initial array's size")
        return ignore_indices.contiguous().reshape(-1).view(torch.uint8)
    mask = np.zeros(shape, dtype=bool)
    mask[ignore_indices] = True
    return _device.to_device(mask.reshape(-1).view(np.uint8))


def _percentile_taps(n, x_wet):
    """(i0, i1, gamma) of np.percentile(target, 100 * (1 - war)) over n sorted values, with
    war = x_wet / n, in NumPy's expressions (numpy/lib/_function_base_impl.py: percentile, _quantile,
    _get_indexes, _get_gamma with method "linear"): the value is _lerp(sorted[i0], sorted[i1], gamma)"""
    war = np.int64(x_wet) / n
    q = np.true_divide(100 * (1 - war), np.float64(100))
    virtual = (n - 1) * q
    if virtual >= n - 1:
        previous = nxt = -1
    else:
        previous = int(np.floor(virtual))
        nxt = previous + 1
    gamma = float(virtual - np.intp(previous))
    return previous % n, nxt % n, gamma


def _scratch(n):
    nbytes = ctypes.c_int64(0)
    _lib.call("b200_pm_scratch_bytes", n, ctypes.byref(nbytes))
    return torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device="cuda")
