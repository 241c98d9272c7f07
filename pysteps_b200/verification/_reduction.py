"""How the deterministic scores reduce over their integration axes: the reference's axis handling, and
NumPy's summation order as a launch plan for the kernels.

The reference integrates over ``axis`` (None: all axes; negative axes are dropped, and when every axis
is negative a leading unit axis is added and reduced, so nothing is integrated).  ``np.sum(a, axis)``
of a C-contiguous float array adds, for every output element, the pairwise sum of the trailing run of
reduced axes (merged into one contiguous run) onto 0, one run after the other over the remaining
reduced axes in C order; size-1 axes do not count.  ``plan`` turns (shape, axis) into that order.
"""
import ctypes

import numpy as np


def kept_shape(shape, axis_opt):
    """(the kept shape as the reference builds it, the axes) of an accumulation over `axis_opt` (the
    dict's "axis"), raising the reference's exceptions"""
    ndim = len(shape)
    axis = tuple(range(ndim)) if axis_opt is None else axis_opt
    if ndim <= np.max(axis):
        raise ValueError("axis %d is out of bounds for array of dimension %d" % (np.max(axis), ndim))
    kept = [d not in axis for d in range(ndim)]
    return tuple(np.array(shape)[np.array(kept)]), axis


def effective(shape, axis):
    """the shape and the non-negative axes the reference reduces; an axis set NumPy rejects raises
    NumPy's exception, replayed on a stand-in"""
    if np.max(axis) < 0:
        shape, axis = (1,) + tuple(shape), (0,)
    axis = tuple(a for a in axis if a >= 0)
    np.sum(np.zeros((1,) * len(shape), dtype=np.int64), axis=axis)
    return tuple(shape), tuple(int(a) for a in axis)


def _strides(shape):
    return [int(np.prod(shape[d + 1:], dtype=np.int64)) for d in range(len(shape))]


def split_axes(shape, axis):
    """((sizes, strides) of the kept axes, (sizes, strides) of the reduced axes) of a C-contiguous
    array, size-1 axes left out, as int64 arrays"""
    st = _strides(shape)
    out = []
    for reduced in (False, True):
        dims = [d for d in range(len(shape)) if (d in axis) == reduced and shape[d] != 1]
        out.append((np.array([shape[d] for d in dims], np.int64), np.array([st[d] for d in dims], np.int64)))
    return out


def plan(shape, axis):
    """NumPy's order of np.sum(a, axis) for a C-contiguous `a` of `shape`: ((sizes, strides) of the
    kept axes, (sizes, strides) of the outer reduced axes, L) -- output element m adds, for every outer
    index in C order, the pairwise sum of the L contiguous elements from offset(m) + offset(outer)"""
    st = _strides(shape)
    dims = [d for d in range(len(shape)) if shape[d] != 1]
    t = len(dims)
    while t > 0 and dims[t - 1] in axis:
        t -= 1
    L = int(np.prod([shape[d] for d in dims[t:]], dtype=np.int64))
    kept = [d for d in dims[:t] if d not in axis]
    outer = [d for d in dims[:t] if d in axis]
    return ((np.array([shape[d] for d in kept], np.int64), np.array([st[d] for d in kept], np.int64)),
            (np.array([shape[d] for d in outer], np.int64), np.array([st[d] for d in outer], np.int64)), L)


def c_axes(sizes, strides):
    """(sizes, strides, count) as the C ABI takes them"""
    p = ctypes.POINTER(ctypes.c_int64)
    return sizes.ctypes.data_as(p), strides.ctypes.data_as(p), len(sizes)
