"""CPU execution of NumPy's pairwise summation as the device runs it: csrc/pairwise_body.cuh, shared
verbatim with csrc/verification.cu, is compiled here as host C++ (into a temporary directory) and must
equal np.sum bit for bit, in float32 and float64, at every length 0-1100, either side of 8192, at
2^16 - 2^20, and for the rows of np.sum(A, axis=1)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
BODY = os.path.join(os.path.dirname(HERE), "pysteps_b200", "csrc", "pairwise_body.cuh")
UNIT = r'''
#include "%s"
extern "C" float pw_f32(const float *x, long long n) {
    auto get = [x](int64_t i) { return x[i]; };
    return pw::pairwise_sum<float, 40>(get, n);
}
extern "C" double pw_f64(const double *x, long long n) {
    auto get = [x](int64_t i) { return x[i]; };
    return pw::pairwise_sum<double, 40>(get, n);
}
'''


@pytest.fixture(scope="module")
def lib():
    with tempfile.TemporaryDirectory() as tmp:
        src, so = os.path.join(tmp, "pw.cpp"), os.path.join(tmp, "libpw.so")
        with open(src, "w") as f:
            f.write(UNIT % BODY)
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-fno-fast-math",
                               "-Wall", "-o", so, src])
        L = ctypes.CDLL(so)
    L.pw_f32.restype, L.pw_f64.restype = ctypes.c_float, ctypes.c_double
    L.pw_f32.argtypes = L.pw_f64.argtypes = [ctypes.c_void_p, ctypes.c_longlong]
    return L


def _sum(L, x):
    fn = L.pw_f32 if x.dtype == np.float32 else L.pw_f64
    return x.dtype.type(fn(x.ctypes.data, len(x)))


def _data(rng, n, dtype):
    return (rng.standard_normal(n) * 10.0 ** rng.uniform(-4, 4, n)).astype(dtype)


LENGTHS = list(range(0, 1101)) + [8190, 8191, 8192, 8193, 8194, 20000, 100003] + [1 << e for e in range(16, 21)] \
    + [(1 << e) + 8 * e + 3 for e in range(16, 20)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pairwise_body_equals_numpy_sum(lib, dtype):
    rng = np.random.default_rng(1)
    bad = [n for n in LENGTHS if _sum(lib, x := _data(rng, n, dtype)).tobytes() != np.sum(x).tobytes()]
    assert not bad, f"lengths differing from np.sum: {bad[:20]}"


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pairwise_body_equals_row_sums(lib, dtype):
    rng = np.random.default_rng(2)
    for cols in (1, 7, 8, 9, 25, 128, 129, 257, 301, 513):
        A = _data(rng, 40 * cols, dtype).reshape(40, cols)
        want = np.sum(A, axis=1)
        got = np.array([_sum(lib, np.ascontiguousarray(r)) for r in A], dtype=dtype)
        assert got.tobytes() == want.tobytes(), cols


def test_all_negative_zeros_sum_to_positive_zero(lib):
    for n in (0, 3, 8, 200):
        x = np.full(n, -0.0)
        assert _sum(lib, x).tobytes() == np.sum(x).tobytes()
