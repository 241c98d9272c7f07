"""TEST INFRASTRUCTURE: the entry points of csrc/probmatching.cu stood in for by the oracle
(oracle/probmatching.py), on top of tests/cpu_abi.py's emulation of the device plumbing, so that the
host logic of pysteps_b200.postprocessing.probmatching runs without a GPU.  The statistics record is
computed here from the data as the kernels define it.

    with cpu_abi_probmatching.emulated():
        out = pysteps_b200.postprocessing.probmatching.nonparam_match_empirical_cdf(a, b)
"""
import contextlib
import ctypes
from unittest import mock

import numpy as np

import cpu_abi
from pysteps_b200 import _lib


def _array(p, code, n):
    return cpu_abi._view(p, (n,), cpu_abi._NP[code]) if n else np.zeros(0, cpu_abi._NP[code])


def _mask(p, n):
    m = cpu_abi._view(p, (n,), np.uint8) if n else None
    return np.zeros(n, bool) if m is None else m.astype(bool)


def _i64(p, n):
    return np.frombuffer((ctypes.c_int64 * n).from_address(cpu_abi._addr(p)), dtype=np.int64)


def _scratch_bytes(n, nbytes):
    ctypes.cast(nbytes, ctypes.POINTER(ctypes.c_int64))[0] = 1


def _match_stats(x, xd, ignore, n_x, t, td, n_t, stats, scratch, nbytes, stream):
    from oracle import probmatching as ora
    X = _array(x, xd, n_x).astype(np.float64)
    T = _array(t, td, n_t).astype(np.float64)
    m = _mask(ignore, n_x)
    zx, zt = ora.signed_nanmin(X), ora.signed_nanmin(T)
    with np.errstate(invalid="ignore"):
        cpu_abi._view(stats, (8,))[:] = [zx, np.count_nonzero(~np.isnan(X)), np.count_nonzero(~np.isfinite(X[~m])),
                                         np.count_nonzero(m), np.count_nonzero(X[~m] > zx), zt,
                                         np.count_nonzero(~np.isnan(T)), np.count_nonzero(T > zt)]


def _match(x, xd, ignore, t, td, n, stats, n_xwet, n_twet, clip, i0, i1, gamma, out, scratch, nbytes, stream):
    from oracle import probmatching as ora
    if n == 0:
        return
    m = _mask(ignore, n)
    X, T = _array(x, xd, n), _array(t, td, n)
    s = cpu_abi._view(stats, (8,))
    assert (n_xwet, n_twet) == (int(s[4]), int(s[7])) and s[2] == 0
    if clip:  # the host's taps are the oracle's
        assert (i0, i1, gamma) == ora.percentile_taps(n, n_xwet)
    cpu_abi._view(out, (n,))[:] = ora.nonparam_match_empirical_cdf(X, T, m)


def _resample_nan(a, ad, b, bd, n, n_nan, stream):
    A, B = _array(a, ad, n), _array(b, bd, n)
    _i64(n_nan, 1)[0] = np.count_nonzero(np.isnan(A) | np.isnan(B))


def _resample(a, ad, b, bd, n, n_nan, draws, out, od, scratch, nbytes, stream):
    from oracle import probmatching as ora
    if n == 0:
        return
    A, B = _array(a, ad, n), _array(b, bd, n)
    r = ora.resample_distributions(A, B, _mask(draws, n))
    assert r.dtype == cpu_abi._NP[od] and np.count_nonzero(np.isnan(r)) == n_nan
    _array(out, od, n)[:] = r


_TABLE = {"b200_pm_scratch_bytes": _scratch_bytes, "b200_pm_match_stats": _match_stats, "b200_pm_match": _match,
          "b200_pm_resample_nan": _resample_nan, "b200_pm_resample": _resample}


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
