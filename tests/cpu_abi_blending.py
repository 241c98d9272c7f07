"""TEST INFRASTRUCTURE: the entry points of csrc/blending.cu stood in for by NumPy (the reference's own
expressions and oracle/blending.py's dense rank), on top of tests/cpu_abi.py's emulation of the rest of
the C ABI (the field statistics and the semi-Lagrangian extrapolator of the extrapolation nowcast), so
that the host logic of pysteps_b200.blending and pysteps_b200.nowcasts.extrapolation runs without a
GPU.  The emulated conversion lists the pixels within the kernel's bound of the threshold, as the
kernel does, so the host's fix-up path runs too.

    with cpu_abi_blending.emulated():
        out = pysteps_b200.blending.get_method("salient_blending")(precip, meta, V, 6, 10, "eulerian", nwp, meta)
"""
import contextlib
import ctypes
from unittest import mock

import numpy as np

import cpu_abi
from oracle import blending as ora
from pysteps_b200 import _lib

_SIZE = {_lib.F32: 4, _lib.F64: 8}
fixups = []  # the number of pixels each emulated conversion left to the host, most recent last


def _i64(p, n):
    return np.frombuffer((ctypes.c_int64 * n).from_address(cpu_abi._addr(p)), dtype=np.int64)


def _plane(ptr, code, offset, P):
    return cpu_abi._view(cpu_abi._addr(ptr) + _SIZE[code] * offset, (P,), cpu_abi._NP[code])


def _transform(x, y, code, n, kind, lam, thr, zero, fix_idx, fix_x, cap, nfix, stream):
    dt = cpu_abi._NP[code]
    count = _i64(nfix, 1) if nfix else None
    if count is not None:
        count[0] = 0
    if n == 0:
        return
    X = cpu_abi._view(x, (n,), dt)
    Y = cpu_abi._view(y, (n,), dt)
    with np.errstate(all="ignore"):
        if kind == 0:
            Y[:] = X
            return
        if kind == 1:
            Y[:] = X * X
            return
        R = [None, None, lambda r: 10.0 ** (r / 10.0), np.exp, lambda r: np.exp(np.log(lam * r + 1) / lam)][kind](X)
        eps = float(np.finfo(dt).eps)
        z = np.abs(np.log(lam * X + 1) / lam).astype(np.float64) if kind == 4 else 0.0
        rel = 16.0 * eps * (2.0 + z) if kind == 4 else 16.0 * eps
        d = R.astype(np.float64)
        near = np.isfinite(d) & (np.abs(d - thr) <= rel * np.maximum(np.abs(d), abs(thr)) + 1e-300)
    out = np.where(~near & (d < thr), dt(zero), R)
    Y[:] = out
    idx = np.flatnonzero(near)
    count[0] = len(idx)
    fixups.append(len(idx))
    k = min(len(idx), cap)
    if k:
        _i64(fix_idx, k)[:] = idx[:k]
        cpu_abi._view(fix_x, (k,))[:] = X[idx[:k]]


def _unit(x, y, code, n, kind, a, b, stream):
    dt = cpu_abi._NP[code]
    if n == 0:
        return
    X = cpu_abi._view(x, (n,), dt)
    with np.errstate(all="ignore"):
        r = X / dt(a) * dt(b) if kind == 1 else (X / dt(a)) ** dt(b)
    cpu_abi._view(y, (n,), dt)[:] = r


def _scatter(y, code, idx, val, n, stream):
    if n:
        i = _i64(idx, n)
        Y = cpu_abi._view(y, (int(i.max()) + 1,), cpu_abi._NP[code])
        Y[i] = cpu_abi._view(val, (n,))


class _Fields:
    def __init__(self, now, cn, now_map, now_member, nwp, cw, nwp_map, nwp_member, n_out, P, fill):
        self.now, self.cn, self.nwp, self.cw = now, cn, nwp, cw
        self.mn = cpu_abi._view(now_map, (n_out,), np.int32)
        self.mw = cpu_abi._view(nwp_map, (n_out,), np.int32)
        self.now_member, self.nwp_member, self.P, self.fill = now_member, nwp_member, P, fill

    def nwp_plane(self, e, i):
        return np.nan_to_num(_plane(self.nwp, self.cw, int(self.mw[e]) * self.nwp_member + i * self.P, self.P))

    def now_plane(self, e, i):
        c = _plane(self.now, self.cn, int(self.mn[e]) * self.now_member + i * self.P, self.P).copy()
        nan = np.isnan(c)
        c[nan] = self.nwp_plane(e, i)[nan] if self.fill else 0.0
        return c


def _linear(now, cn, now_map, now_member, nwp, cw, nwp_map, nwp_member, out, n_out, T, P, mode, bits, w_nwp, w_now,
            fill, stream):
    f = _Fields(now, cn, now_map, now_member, nwp, cw, nwp_map, nwp_member, n_out, P, fill)
    md, bt = cpu_abi._view(mode, (T,), np.int32), cpu_abi._view(bits, (T,), np.int32)
    wn, wc = cpu_abi._view(w_nwp, (T,)), cpu_abi._view(w_now, (T,))
    for e in range(n_out):
        for i in range(T):
            o = _plane(out, cw, (e * T + i) * P, P)
            if md[i] == 0:
                o[:] = f.now_plane(e, i)
            elif md[i] == 1:
                o[:] = f.nwp_plane(e, i)
            elif md[i] == 2:
                g, c = f.nwp_plane(e, i), f.now_plane(e, i)
                a = wn[i] * g.astype(np.float64) if bt[i] & 1 else g.dtype.type(wn[i]) * g
                b = wc[i] * c.astype(np.float64) if bt[i] & 2 else c.dtype.type(wc[i]) * c
                o[:] = a.astype(np.float64) + b if bt[i] & 4 else np.float32(a) + np.float32(b)


def _salient(now, cn, now_map, now_member, nwp, cw, nwp_map, nwp_member, out, n_out, T, P, lead, w, w1, w2, w12, fill,
             scratch, nbytes, stream):
    f = _Fields(now, cn, now_map, now_member, nwp, cw, nwp_map, nwp_member, n_out, P, fill)
    c = np.stack([f.now_plane(e, lead) for e in range(n_out)])
    g = np.stack([f.nwp_plane(e, lead) for e in range(n_out)])
    with np.errstate(all="ignore"):
        nc = np.zeros_like(c) if np.max(c) == 0 else c / np.max(c)
        ng = np.zeros_like(g) if np.max(g) == 0 else g / np.max(g)
        r = ora.dense_rank(nc - ng).reshape(c.shape)
        r /= r.max()
        s1 = np.sqrt(r * r + w2)
        ws = 0.5 * ((w * r) / (w * r + w1 * (1 - r)) + s1 / (s1 + np.sqrt((1 - r) * (1 - r) + w12)))
        v = ws * c + (1 - ws) * g
    for e in range(n_out):
        _plane(out, cw, (e * T + lead) * P, P)[:] = v[e]


def _scratch_bytes(n, out):
    out._obj.value = 1  # ctypes.byref(c_int64)


_TABLE = {"b200_blend_transform": _transform, "b200_blend_unit": _unit, "b200_blend_scatter": _scatter,
          "b200_blend_linear": _linear, "b200_blend_salient": _salient, "b200_blend_scratch_bytes": _scratch_bytes}


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
