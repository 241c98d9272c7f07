"""B200 constant advection field -- drop-in for ``pysteps.motion.constant.constant``
(pysteps/motion/constant.py:20-54): the translation that maximises the correlation of the last two
frames.  scipy's Nelder-Mead runs on the host with the reference's arguments; every point it visits
is one ``b200_constant_eval`` call (csrc/constant.cu) and a 24-byte read-back of its record.

The objective is the reference's at every point: the same counted pixels, NumPy's pairwise means
bit for bit and NumPy's corrcoef tail; only the three centred sums, which the reference forms with
a BLAS dot product, are summed in a fixed order of the kernel's.  The reference's RuntimeWarnings
(empty overlap, fewer than two pixels, constant overlaps) are raised from the record's bits, by the
same NumPy operations, so ``np.errstate`` and warning filters act on them as on the reference's.

Parity: tests/test_constant_gpu.py (device), tests/test_oracle_constant.py and
tests/test_host_logic_constant.py (oracle and host logic on the CPU).
"""
import warnings

import numpy as np
import scipy.optimize as op
import torch

from .. import _device, _lib

# the B200_CONST_* bits of include/pysteps_b200.h
_EMPTY, _DOF, _SCALE_INVALID = 1, 2, 4
_ROW_BITS, _COL_BITS = (8, 16, 32), (64, 128, 256)  # invalid, divide by zero, overflow


def _divide_events(bits):
    """np.true_divide on operands that raise exactly these events (one warning per kind, numpy's order)."""
    x, y = [], []
    for bit, (a, b) in zip(bits, ((0.0, 0.0), (1.0, 0.0), (1e308, 1e-308))):
        if bit:
            x.append(a)
            y.append(b)
    if x:
        np.true_divide(np.array(x), np.array(y))


def _raise_warnings(flags):
    """The RuntimeWarnings of np.corrcoef (np.cov, np.mean) for one evaluation, in their order."""
    if flags & _EMPTY:
        warnings.warn("Mean of empty slice.", RuntimeWarning, stacklevel=3)
        np.true_divide(np.zeros(2), 0)
    if flags & _DOF:
        warnings.warn("Degrees of freedom <= 0 for slice", RuntimeWarning, stacklevel=3)
        np.true_divide(1, 0.0)
    if flags & _SCALE_INVALID:
        np.multiply(np.zeros(1), np.inf)
    _divide_events([flags & b for b in _ROW_BITS])
    _divide_events([flags & b for b in _COL_BITS])


def constant(R, **kwargs):
    """Same contract as the reference (constant.py:20-37): R (T, m, n), T >= 2, the last two frames
    are used, kwargs are ignored.  NumPy input (a MaskedArray is used through its data, as the
    reference's map_coordinates and corrcoef see it) -> NumPy (2, m, n) float64; CUDA tensor input
    (NaN = no data) -> a (2, m, n) float64 tensor on the same device."""
    m, n = R.shape[1:]
    on_device = _device.is_device_tensor(R)
    if isinstance(R, np.ma.MaskedArray):
        R = np.ma.getdata(R)
    # the reference fails on R[-2] at its first evaluation when there is one frame
    prev, nxt = R[-2], R[-1]
    lib = torch if isinstance(prev, torch.Tensor) else np
    if prev.dtype == lib.float16:
        raise RuntimeError("data type not supported")  # scipy's map_coordinates
    if prev.dtype not in (lib.float32, lib.float64):
        raise NotImplementedError(f"pysteps_b200 constant: frames of dtype {prev.dtype} are not supported "
                                  "(float32 or float64)")
    m, n = int(m), int(n)

    _device.require_cuda()
    d_prev, d_next = _device.to_device(prev), _device.to_device(nxt)
    code = _device.dtype_code(d_prev.dtype)
    nbytes = _lib.c_i64(0)
    _lib.call("b200_constant_scratch_bytes", m, n, nbytes)
    scratch = torch.zeros(int(nbytes.value), dtype=torch.uint8, device="cuda")
    record = torch.empty(3, dtype=torch.float64, device="cuda")
    host = torch.empty(3, dtype=torch.float64, pin_memory=True)
    done = torch.cuda.Event()

    def f(v):
        _lib.call("b200_constant_eval", d_prev.data_ptr(), d_next.data_ptr(), code, m, n, float(v[0]),
                  float(v[1]), scratch.data_ptr(), record.data_ptr(), _device.stream_ptr())
        host.copy_(record, non_blocking=True)
        done.record()
        done.synchronize()
        value, _count, flags = host.tolist()
        _raise_warnings(int(flags))
        return np.float64(value)

    options = {"initial_simplex": (np.array([(0, 1), (1, 0), (1, 1)]))}
    result = op.minimize(f, (1, 1), method="Nelder-Mead", options=options)

    ux, uy = -result.x[0], -result.x[1]
    if not on_device:
        out = np.empty((2, m, n))  # the bits of np.stack([ux * np.ones((m, n)), uy * np.ones((m, n))])
        out[0] = ux
        out[1] = uy
        return out
    out = torch.empty((2, m, n), dtype=torch.float64, device="cuda")
    for c, u in enumerate((ux, uy)):
        if m * n:
            _lib.call("b200_fill_f64", out[c].data_ptr(), m * n, float(u), _device.stream_ptr())
    return out
