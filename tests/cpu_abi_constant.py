"""TEST INFRASTRUCTURE: the two entry points of csrc/constant.cu stood in for by the oracle
(oracle/constant.py, which restates the kernels' order), on top of tests/cpu_abi.py's emulation of
the rest of the C ABI, so that the host logic of pysteps_b200.motion.constant runs without a GPU.

    with cpu_abi_constant.emulated():
        field = pysteps_b200.motion.get_method("constant")(R)
"""
import contextlib
from unittest import mock

import numpy as np

import cpu_abi
from pysteps_b200 import _lib


def _scratch_bytes(m, n, nbytes):
    nbytes.value = 8


def _eval(prev, nxt, code, m, n, vx, vy, scratch, record, stream):
    from oracle import constant as ora_constant
    dt = cpu_abi._NP[code]
    frames = [cpu_abi._view(p, (m, n), dt) if m * n else np.empty((m, n), dt) for p in (prev, nxt)]
    f, count, flags = ora_constant.evaluate(frames[0], frames[1], vx, vy)
    cpu_abi._view(record, (3,))[...] = (f, count, flags)


_TABLE = {"b200_constant_scratch_bytes": _scratch_bytes, "b200_constant_eval": _eval}


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
