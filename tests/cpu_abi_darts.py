"""TEST INFRASTRUCTURE: the three entry points of csrc/darts.cu stood in for by the oracle
(oracle/darts.py), on top of tests/cpu_abi.py's emulation of the rest of the C ABI, so that the host
logic of pysteps_b200.motion.darts runs without a GPU.

    with cpu_abi_darts.emulated():
        field = pysteps_b200.motion.get_method("darts")(R, verbose=False)
"""
import contextlib
from unittest import mock

import numpy as np

import cpu_abi
from pysteps_b200 import _lib


def _cview(p, shape):
    """complex128 view of an interleaved (re, im) float64 buffer"""
    return cpu_abi._view(p, tuple(shape[:-1]) + (2 * shape[-1],)).view(np.complex128)


def _spectrum(frames, code, T, m, n, tw_x, fx, tw_y, Ky, tw_t, Kt, K, work, out, stream):
    from oracle import darts as ora
    R = cpu_abi._view(frames, (T, m, n), cpu_abi._NP[code])
    X = ora.spectrum_from_tables(R, _cview(tw_x, (fx, n)), _cview(tw_y, (Ky, m)), _cview(tw_t, (Kt, T)), K)
    _cview(out, (Kt, Ky, 2 * K + 1))[...] = X


def _normal(spec, N_x, N_y, N_t, M_x, M_y, sx, sy, work, mm, mhy, stream):
    from oracle import darts as ora
    X = _cview(spec, (2 * N_t + 1, 2 * (N_y + M_y) + 1, 2 * (N_x + M_x) + 1))
    nc = 2 * (2 * M_x + 1) * (2 * M_y + 1)
    MM, Mhy = ora.normal(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    _cview(mm, (nc, nc))[...] = MM
    _cview(mhy, (nc,))[...] = Mhy


def _synthesize(coef, h, w, ey, ex, m, n, out, stream):
    from oracle import darts as ora
    cpu_abi._view(out, (2, m, n))[...] = ora.synthesize(_cview(coef, (2, h, w)), _cview(ey, (h, m)),
                                                        _cview(ex, (w, n)), m, n)


_TABLE = {"b200_darts_spectrum": _spectrum, "b200_darts_normal": _normal, "b200_darts_synthesize": _synthesize}


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
