"""TEST INFRASTRUCTURE: the entry points of csrc/detscores.cu and csrc/fss.cu stood in for by NumPy and
the oracle (oracle/detscores.py), on top of tests/cpu_abi.py's emulation of the device, so that the
host logic of pysteps_b200.verification's deterministic and spatial scores runs without a GPU.
Numerically this checks the host code only; the kernels are checked by tests/test_detscores_gpu.py.

    with cpu_abi_detscores.emulated():
        out = pysteps_b200.verification.fss(X_f, X_o, 1.0, 16)
"""
import contextlib
from unittest import mock

import numpy as np

import cpu_abi
from cpu_abi_verification import _arr, _np
from oracle import detscores as ora
from oracle.verification import pairwise
from pysteps_b200 import _lib


def _host(p, n):
    return np.array([p[i] for i in range(n)], dtype=np.int64)


def _contab(pred, pd, obs, od, thr_p, thr_o, ks, kst, nk, rs, rst, nr, counts, stream):
    ks, kst, rs, rst = _host(ks, nk), _host(kst, nk), _host(rs, nr), _host(rst, nr)
    M, R = int(np.prod(ks)), int(np.prod(rs))
    off = np.zeros(1, np.int64)
    for size, stride in zip(ks, kst):
        off = (off[:, None] + np.arange(size) * stride).reshape(-1)
    roff = np.zeros(1, np.int64)
    for size, stride in zip(rs, rst):
        roff = (roff[:, None] + np.arange(size) * stride).reshape(-1)
    idx = off[:, None] + roff[None, :]
    total = int(idx.max()) + 1 if idx.size else 0
    p = _arr(pred, total, _np(pd)).astype(np.float64)[idx] > thr_p
    o = _arr(obs, total, _np(od)).astype(np.float64)[idx] > thr_o
    out = _arr(counts, 4 * M, np.int64).reshape(4, M)
    for j, c in enumerate((p & o, p & ~o, ~p & o, ~p & ~o)):
        out[j] = c.reshape(M, R).sum(axis=1)


def _offsets(sizes, strides):
    off = np.zeros(1, np.int64)
    for size, stride in zip(sizes, strides):
        off = (off[:, None] + np.arange(size) * stride).reshape(-1)
    return off


def _bits(v, k):
    return np.where(np.isposinf(v), 1 << (2 * k), 0) | np.where(np.isneginf(v), 1 << (2 * k + 1), 0)


def _op(r, a, b, over, inv):
    f = over if (np.isinf(r) & np.isfinite(a) & np.isfinite(b)).any() else 0
    return f | (inv if (np.isnan(r) & ~np.isnan(a) & ~np.isnan(b)).any() else 0)


def _moments(pred, pd, obs, od, cond, thr_p, thr_o, ks, kst, nk, os_, ost, no, L, tot, cnt, infs, flags, stream):
    """b200_verif_cont_moments: the runs of the host's plan, each summed pairwise (the oracle's
    restatement), added onto 0 in order"""
    base = _offsets(_host(ks, nk), _host(kst, nk))
    outer = _offsets(_host(os_, no), _host(ost, no))
    idx = base[:, None, None] + outer[None, :, None] + np.arange(L)[None, None, :]
    P, Q = _np(pd), _np(od)
    R = np.result_type(P, Q)
    p = _arr(pred, int(idx.max()) + 1, P)[idx]
    q = _arr(obs, int(idx.max()) + 1, Q)[idx]
    if cond:
        sp, so = p.astype(np.float64) > thr_p, q.astype(np.float64) > thr_o
        keep = (sp | so) if cond == 1 else (sp & so)
        p, q = np.where(keep, p, np.nan).astype(P), np.where(keep, q, np.nan).astype(Q)
    M = len(base)
    t, c = _arr(tot, 9 * M, np.float64).reshape(9, M), _arr(cnt, 10 * M, np.int64).reshape(10, M)
    bits = np.zeros(M, np.int32)
    fl = 0

    def add(k, v):
        nonlocal bits
        z = np.where(np.isnan(v), v.dtype.type(0), v)
        part = pairwise(np.ascontiguousarray(z))
        acc = np.zeros(M, v.dtype)
        for o in range(part.shape[1]):
            acc = acc + part[:, o]
        t[k] = acc
        c[1 + k] = (~np.isnan(v)).sum(axis=(1, 2))
        bits |= np.bitwise_or.reduce(_bits(v, k).reshape(M, -1), axis=1).astype(np.int32)
        return acc

    with np.errstate(all="ignore"):
        rp, rq = p.astype(R), q.astype(R)
        r, sm = rp - rq, rp + rq
        fl |= _op(r, rp, rq, _lib.MOM_SUB_RES_OVER, _lib.MOM_SUB_RES_INV)
        fl |= _op(sm, rp, rq, _lib.MOM_ADD_SUM_OVER, _lib.MOM_ADD_SUM_INV)
        fl |= _op(r * r, r, r, _lib.MOM_SQ_RES_OVER, 0) | _op(sm * sm, sm, sm, _lib.MOM_SQ_SUM_OVER, 0)
        c[0] = np.isfinite(r).sum(axis=(1, 2))
        to, tp = add(0, q), add(1, p)
        for k, v in ((2, r), (3, r * r), (4, sm * sm), (5, np.abs(r))):
            add(k, v)
        mo = (to.astype(np.float64) / c[1]).astype(Q)[:, None, None]
        mp = (tp.astype(np.float64) / c[2]).astype(P)[:, None, None]
        x, y = q - mo, p - mp
        cv = x.astype(R) * y.astype(R)
        fl |= _op(x, q, np.broadcast_to(mo, q.shape), _lib.MOM_SUB_OBS_OVER, _lib.MOM_SUB_OBS_INV)
        fl |= _op(y, p, np.broadcast_to(mp, p.shape), _lib.MOM_SUB_PRED_OVER, _lib.MOM_SUB_PRED_INV)
        fl |= _op(cv, x, y, _lib.MOM_MUL_OVER, _lib.MOM_MUL_INV)
        vx, vy = np.abs(x) * np.abs(x), np.abs(y) * np.abs(y)
        fl |= _op(vx, x, x, _lib.MOM_SQ_VOBS_OVER, 0) | _op(vy, y, y, _lib.MOM_SQ_VPRED_OVER, 0)
        for k, v in ((6, cv), (7, vx), (8, vy)):
            add(k, v)
    _arr(infs, M, np.int32)[:] = bits
    _arr(flags, 1, np.int32)[0] = fl


def _fractions(X, dtype, nf, m, n, thr, sub, s, S, stream):
    x = _arr(X, nf * m * n, _np(dtype)).reshape(nf, m, n).astype(np.float64)
    I = (np.where(np.isfinite(x), x, sub) >= thr).astype(np.float64)
    out = _arr(S, nf * m * n, np.float64).reshape(nf, m, n)
    for f in range(nf):
        out[f] = I[f] if s <= 1 else ora.uniform_filter(I[f], s)


def _sums(S, P, a0, na, b0, nb, out, stream):
    planes = _arr(S, (max(a0 + na, b0 + nb)) * P, np.float64).reshape(-1, P)
    o = _arr(out, na * nb, np.float64).reshape(na, nb)
    for i in range(na):
        for j in range(nb):
            if a0 + i <= b0 + j:
                o[i, j] = pairwise(planes[a0 + i] * planes[b0 + j])


_TABLE = {"b200_verif_contab": _contab, "b200_verif_cont_moments": _moments, "b200_fss_fractions": _fractions,
          "b200_fss_sums": _sums}


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
