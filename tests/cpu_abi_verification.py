"""TEST INFRASTRUCTURE: the entry points of csrc/verification.cu stood in for by NumPy and the oracle
(oracle/verification.py), on top of tests/cpu_abi.py's emulation of the device, so that the host logic
of pysteps_b200.verification runs without a GPU.  Numerically this checks the host code only; the
kernels are checked by tests/test_verification_gpu.py.

    with cpu_abi_verification.emulated():
        crps = pysteps_b200.verification.probscores.CRPS(X_f, X_o)
"""
import contextlib
import ctypes
from unittest import mock

import numpy as np

import cpu_abi
from oracle import verification as ora
from pysteps_b200 import _lib


def _arr(p, n, dtype):
    a = cpu_abi._addr(p)
    if a is None or n == 0:
        return np.zeros(n, dtype)
    ct = {np.int64: ctypes.c_int64, np.int32: ctypes.c_int32, np.float32: ctypes.c_float,
          np.float64: ctypes.c_double}[dtype]
    return np.frombuffer((ct * n).from_address(a), dtype=dtype)


def _np(code):
    return cpu_abi._NP[code]


def _crps(Xf, fd, Xo, od, k, N, res, n, stream):
    per = ora.crps_pixels(_arr(Xf, k * N, _np(fd)).reshape(k, N), _arr(Xo, N, _np(od)))
    _arr(res, len(per), np.float64)[:] = per
    _arr(n, 1, np.int64)[0] = len(per)


def _pairwise(x, dtype, seg_off, seg_len, nseg, out, stream):
    off = _arr(seg_off, nseg, np.int64)
    ln = _arr(seg_len, nseg, np.int64)
    total = int((off + ln).max()) if nseg else 0
    v = _arr(x, total, _np(dtype))
    o = _arr(out, nseg, _np(dtype))
    for s in range(nseg):
        o[s] = ora.pairwise(np.ascontiguousarray(v[off[s]:off[s] + ln[s]]))


def _rankhist(Xf, fd, Xo, od, k, N, use_min, thr_f, sub_f, thr_o, sub_o, hist, ties, n_ties, stream):
    F = _arr(Xf, k * N, _np(fd)).reshape(k, N).astype(np.float64)
    O = _arr(Xo, N, _np(od)).astype(np.float64)
    keep = np.isfinite(F).all(axis=0) & np.isfinite(O)
    if use_min:
        keep &= (O >= thr_o) | (F >= thr_f).any(axis=0)
        F = np.where(F < thr_f, sub_f, F)
        O = np.where(O < thr_o, sub_o, O)
    F, O = F[:, keep], O[keep]
    b1 = (F < O).sum(axis=0)
    b2 = k - (F > O).sum(axis=0)
    tied = (F == O).any(axis=0)
    _arr(hist, k + 1, np.int64)[:] = np.bincount(b1[~tied], minlength=k + 1)
    pairs = np.stack([b1[tied], b2[tied]], axis=1).astype(np.int32).reshape(-1)
    _arr(ties, len(pairs), np.int32)[:] = pairs
    _arr(n_ties, 1, np.int64)[0] = int(tied.sum())


def _rankhist_ties(ties, n_ties, u, k, hist, stream):
    pairs = _arr(ties, 2 * n_ties, np.int32).reshape(n_ties, 2).astype(np.int64)
    bins = (pairs[:, 0] + _arr(u, n_ties, np.float64) * (pairs[:, 1] + 1 - pairs[:, 0])).astype(np.int64)
    _arr(hist, k + 1, np.int64)[:] += np.bincount(bins, minlength=k + 1)


def _reldiag(P, pd, Xo, od, N, edges, n_edges, thr_o, sorted_, seg, above, stream):
    p = _arr(P, N, _np(pd))
    o = _arr(Xo, N, _np(od)).astype(np.float64)
    e = np.array([edges[i] for i in range(n_edges)])
    nb = n_edges - 1
    keep = np.isfinite(p) & np.isfinite(o)
    b = np.where(keep, (p.astype(np.float64)[:, None] > e[None, :]).sum(axis=1), -1)
    inside = (b >= 1) & (b <= nb)
    order = np.argsort(np.where(inside, b, nb + 1), kind="stable")[:int(inside.sum())]
    _arr(sorted_, len(order), _np(pd))[:] = p[order]
    counts = np.bincount(b[inside] - 1, minlength=nb) if nb else np.zeros(0, np.int64)
    _arr(seg, n_edges, np.int64)[:] = np.concatenate([[0], np.cumsum(counts)])
    if nb:
        _arr(above, nb, np.int64)[:] = np.bincount(b[inside & (o >= thr_o)] - 1, minlength=nb)


def _roc(P, pd, Xo, od, N, thr, n_thr, thr_o, counts, stream):
    p = _arr(P, N, _np(pd)).astype(np.float64)
    o = _arr(Xo, N, _np(od)).astype(np.float64)
    t = np.array([thr[i] for i in range(n_thr)])
    keep = np.isfinite(p) & np.isfinite(o)
    c = (p[keep][:, None] >= t[None, :]).sum(axis=1)
    ev = o[keep] >= thr_o
    out = _arr(counts, 2 * (n_thr + 1), np.int64)
    out[:n_thr + 1] = np.bincount(c[ev], minlength=n_thr + 1)
    out[n_thr + 1:] = np.bincount(c[~ev], minlength=n_thr + 1)


_TABLE = {"b200_verif_crps": _crps, "b200_pairwise_sum": _pairwise, "b200_verif_rankhist": _rankhist,
          "b200_verif_rankhist_ties": _rankhist_ties, "b200_verif_reldiag": _reldiag, "b200_verif_roc": _roc}


@contextlib.contextmanager
def emulated():
    with cpu_abi.emulated():
        rest = _lib.call

        def call(name, *args):
            if name in _TABLE:
                return _TABLE[name](*args)
            return rest(name, *args)

        with mock.patch.object(_lib, "call", call):
            yield
