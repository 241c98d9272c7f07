"""Input handling shared by the verification scores: which arrays the device takes, how they reach it,
and the reference's own exceptions for shapes it cannot use."""
import numpy as np
import torch

from .. import _compare, _device, _lib


def check(a, who, name):
    """a NumPy array or a CUDA tensor of float32 or float64, with fewer than 2^31 pixels per member"""
    if isinstance(a, torch.Tensor):
        if not a.is_cuda:
            raise NotImplementedError(f"pysteps_b200 {who}: {name} must be a NumPy array or a CUDA tensor")
        ok = a.dtype in (torch.float32, torch.float64)
    elif isinstance(a, np.ndarray):
        if isinstance(a, np.ma.MaskedArray):
            raise NotImplementedError(f"pysteps_b200 {who}: masked arrays are not supported")
        ok = a.dtype in (np.float32, np.float64)
    else:
        raise NotImplementedError(f"pysteps_b200 {who}: {name} must be a NumPy array or a CUDA tensor")
    if not ok:
        raise NotImplementedError(f"pysteps_b200 {who}: {name} of dtype {a.dtype} is not supported "
                                  "(float32 or float64)")


def np_dtype(a):
    return np.dtype(np.float32) if a.dtype in (np.float32, torch.float32) else np.dtype(np.float64)


def pixels(shape):
    return int(np.prod(shape, dtype=np.int64))


def check_pixels(N, who):
    if N >= 1 << 31:
        raise NotImplementedError(f"pysteps_b200 {who}: 2^31 pixels or more per member are not supported")


def check_members(k, who):
    if k > _lib.VERIF_MAX_MEMBERS:
        raise NotImplementedError(f"pysteps_b200 {who}: more than {_lib.VERIF_MAX_MEMBERS} members are not "
                                  "supported")


def threshold(dtype, thr, who):
    """thr as the float64 the kernels compare a field of `dtype` with (NumPy's NEP 50 dtype)"""
    if not isinstance(thr, (int, float, np.integer, np.floating)) or isinstance(thr, bool):
        if not (isinstance(thr, np.ndarray) and thr.ndim == 0 and thr.dtype.kind in "iuf"):
            raise NotImplementedError(f"pysteps_b200 {who}: thresholds must be real scalars")
    return _compare.comparison_threshold(dtype, thr, who)[0]


def to_device(a, shape):
    """a as a C-contiguous device tensor of its own dtype, reshaped to `shape`"""
    _device.require_cuda()
    d = a.contiguous() if isinstance(a, torch.Tensor) else _device.to_device(np.ascontiguousarray(a))
    return d.reshape(shape)


def _dummy(shape):
    return np.zeros(shape, dtype=bool)


def ensemble_shapes(f_shape, o_shape, obs_first=False):
    """How the reference lays out an ensemble of shape f_shape and observations of shape o_shape as
    (pixels, members) and (pixels,): True when every pixel pairs up, "empty" when the reference goes on
    with no pixel at all (NumPy lets an empty boolean mask index a length-1 axis), False otherwise.
    Shapes the reference rejects raise its exception, replayed on boolean stand-ins (obs_first: the
    mask is built observation first, as rankhist builds it)."""
    if len(f_shape) >= 2 and f_shape[0] > 0 and pixels(o_shape) == pixels(f_shape[1:]):
        return True
    X_f, X_o = _dummy(f_shape), _dummy(o_shape)
    X_f = np.vstack([X_f[i, :].flatten() for i in range(X_f.shape[0])]).T
    X_o = X_o.flatten()
    mask = np.logical_and(X_o, np.all(X_f, axis=1)) if obs_first else np.logical_and(np.all(X_f, axis=1), X_o)
    X_f[mask, :], X_o[mask]
    return "empty" if mask.size == 0 else False


def pair_shapes(p_shape, o_shape):
    """The same for the element-wise pairs of reldiag and the ROC curve"""
    if tuple(p_shape) == tuple(o_shape):
        return True
    P, O = _dummy(p_shape), _dummy(o_shape)
    mask = np.logical_and(P, O)
    P[mask], O[mask]
    return "empty" if mask.size == 0 else False


def empty(a, shape):
    """an empty array or tensor of a's kind and dtype"""
    if isinstance(a, torch.Tensor):
        return torch.zeros(shape, dtype=a.dtype, device=a.device)
    return np.zeros(shape, dtype=a.dtype)
