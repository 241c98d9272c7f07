"""TEST INFRASTRUCTURE: the entry point of csrc/probability.cu stood in for by the oracle
(oracle/probability.py, exact int64 counts), on top of tests/cpu_abi.py's emulation of the rest of
the C ABI (the extrapolator and the field statistics), so that the host logic of
pysteps_b200.nowcasts.lagrangian_probability runs without a GPU.  The emulation also checks that
the run table the host uploads is the oracle's kernel.

    with cpu_abi_probability.emulated():
        P = pysteps_b200.nowcasts.get_method("probability")(precip, velocity, 6, 1.0)
"""
import contextlib
from unittest import mock

import numpy as np
import torch

import cpu_abi
from pysteps_b200 import _device, _lib


def _probability(field, code, plane_stride, T, m, n, threshold, nan_exceeds, scales, runs, scratch, out, stream):
    from oracle import probability as ora
    dt = cpu_abi._NP[code]
    S = [int(scales[t]) for t in range(T)]
    table = cpu_abi._view(runs, (sum(S), 2), np.int32) if sum(S) else np.empty((0, 2), np.int32)
    o = cpu_abi._view(out, (T, m, n))
    at = 0
    for t, s in enumerate(S):
        assert np.array_equal(table[at:at + s], ora.kernel_runs(s)), s
        at += s
        addr = cpu_abi._addr(field) + t * plane_stride * np.dtype(dt).itemsize
        F = np.frombuffer((cpu_abi._C[dt] * (m * n)).from_address(addr), dtype=dt).reshape(m, n)
        valid = ~np.isnan(F)
        with np.errstate(invalid="ignore"):
            B = np.where(valid, F.astype(np.float64) >= threshold, bool(nan_exceeds))
        o[t] = ora.neighbourhood(B, valid, s)


@contextlib.contextmanager
def emulated():
    with cpu_abi.emulated():
        rest = _lib.call  # cpu_abi's dispatcher

        def call(name, *args):
            if name == "b200_probability":
                return _probability(*args)
            return rest(name, *args)

        # the stand-in device tensors are host tensors: the extrapolator must hand its field back as
        # a tensor, as it does on the device, for the nowcast to keep it
        with mock.patch.object(_lib, "call", call), \
                mock.patch.object(_device, "is_device_tensor", lambda x: isinstance(x, torch.Tensor)):
            yield

