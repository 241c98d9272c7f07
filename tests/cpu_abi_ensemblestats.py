"""TEST INFRASTRUCTURE: the entry points of csrc/ensemblestats.cu stood in for by the oracle
(oracle/ensemblestats.py), on top of tests/cpu_abi.py's emulation of the rest of the C ABI (the field
statistics behind banddepth's nanmin), so that the host logic of
pysteps_b200.postprocessing.ensemblestats runs without a GPU.  The flags the kernels report are
computed here from the data, with NumPy's own floating-point checks.

    with cpu_abi_ensemblestats.emulated():
        P = pysteps_b200.postprocessing.get_method("excprob", "ensemblestats")(X, 1.0)
"""
import contextlib
import ctypes
import warnings
from unittest import mock

import numpy as np

import cpu_abi
from pysteps_b200 import _lib

_OVERFLOW, _INVALID, _EMPTY = 1, 2, 4


def _i64(p, n):
    return np.frombuffer((ctypes.c_int64 * n).from_address(cpu_abi._addr(p)), dtype=np.int64)


def _members(X, code, k, N):
    return cpu_abi._view(X, (k, N), cpu_abi._NP[code]) if k and N else np.zeros((k, N), cpu_abi._NP[code])


def _sum_flags(V):
    """the flags of the sequential sum over the rows of V, from NumPy's own floating-point status"""
    fl = 0
    acc = np.zeros(V.shape[1:], dtype=V.dtype)
    for i in range(V.shape[0]):
        with warnings.catch_warnings(), np.errstate(over="raise", invalid="ignore"):
            try:
                np.add(acc, V[i])
            except FloatingPointError:
                fl |= _OVERFLOW
        with np.errstate(all="ignore"):
            s = acc + V[i]
        if (np.isnan(s) & ~np.isnan(acc) & ~np.isnan(V[i])).any():
            fl |= _INVALID
        acc = s
    return fl


def _mean(X, code, k, N, nan_mode, use_thr, thr, out, flags, stream):
    from oracle import ensemblestats as ora
    V = _members(X, code, k, N)
    flag = cpu_abi._view(flags, (1,), np.int32)
    flag[0] = 0
    if N == 0:
        return
    o = cpu_abi._view(out, (N,), cpu_abi._NP[code])
    if nan_mode:
        thr_arg = np.float64(thr) if use_thr else None
        o[:] = ora.mean(V[:, None], ignore_nan=True, X_thr=thr_arg)[0]
        drop = np.isnan(V) | ((V.astype(np.float64) < thr) if use_thr else False)
        flag[0] = _sum_flags(np.where(drop, V.dtype.type(0), V)) | (_EMPTY if (~drop).sum(axis=0).min() == 0 else 0)
    else:
        o[:] = ora.mean(V[:, None])[0]
        flag[0] = _sum_flags(V)


def _excprob(X, code, k, N, thr, n_thr, ignore_nan, out, flags, stream):
    from oracle import ensemblestats as ora
    V = _members(X, code, k, N)
    flag = cpu_abi._view(flags, (1,), np.int32)
    flag[0] = 0
    if N == 0 or n_thr == 0:
        return
    t = [np.float64(thr[i]) for i in range(n_thr)]  # already rounded to the comparison dtype
    o = cpu_abi._view(out, (n_thr, N))
    o[:] = ora.excprob(V.astype(np.float64), t, ignore_nan=bool(ignore_nan))
    if ignore_nan and np.isfinite(V).sum(axis=0).min() == 0:
        flag[0] = _EMPTY


def _band_mask(X, code, k, N, thr, col, p, stream):
    from oracle import ensemblestats as ora
    d_p = _i64(p, 1)
    if N == 0:
        d_p[0] = 0
        return
    mask, c = ora.band_mask(_members(X, code, k, N).astype(np.float64), np.float64(thr))
    cpu_abi._view(col, (N,), np.int32)[:] = c
    d_p[0] = int(mask.sum())


def _band_match(X, code, k, N, col, b, p, match, stream):
    from oracle import ensemblestats as ora
    if k == 0:
        return
    m = _i64(match, k)
    if p == 0:
        m[:] = 0
        return
    c = cpu_abi._view(col, (N,), np.int32)
    m[:] = ora.band_match(_members(X, code, k, N), c >= 0, cpu_abi._view(b, (k, p)))


_TABLE = {"b200_ensemble_mean": _mean, "b200_ensemble_excprob": _excprob, "b200_ensemble_band_mask": _band_mask,
          "b200_ensemble_band_match": _band_match}


@contextlib.contextmanager
def emulated():
    with cpu_abi.emulated():
        rest = _lib.call  # cpu_abi's dispatcher

        def call(name, *args):
            if name in _TABLE:
                return _TABLE[name](*args)
            return rest(name, *args)

        with mock.patch.object(_lib, "call", call):
            yield
