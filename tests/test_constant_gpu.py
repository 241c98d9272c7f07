"""GPU: the constant advection method (csrc/constant.cu behind motion/constant.py) against the
reference's recorded runs (tests/golden/constant_golden.npz) and the oracle (oracle/constant.py)."""
import os
import warnings

import numpy as np
import pytest

from constant_cases import CASES, ORDER_DECIDED, build_case
from oracle import constant as ora

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "constant_golden.npz")


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


def _same(a, b):
    """bit for bit, any NaN equal to any NaN"""
    return (np.isnan(a) and np.isnan(b)) or _bits(a) == _bits(b)


def _field(x, m, n):
    return np.stack([-x[0] * np.ones((m, n)), -x[1] * np.ones((m, n))])


class _Evaluator:
    """b200_constant_eval on device copies of two frames, read back after every call."""

    def __init__(self, prev, nxt):
        import torch
        from pysteps_b200 import _device, _lib
        _device.require_cuda()
        self.torch, self.lib, self.dev = torch, _lib, _device
        self.prev, self.next = _device.to_device(prev), _device.to_device(nxt)
        self.m, self.n = prev.shape
        nbytes = _lib.c_i64(0)
        _lib.call("b200_constant_scratch_bytes", self.m, self.n, nbytes)
        self.scratch = torch.zeros(int(nbytes.value), dtype=torch.uint8, device="cuda")
        self.record = torch.empty(3, dtype=torch.float64, device="cuda")

    def __call__(self, vx, vy):
        self.lib.call("b200_constant_eval", self.prev.data_ptr(), self.next.data_ptr(),
                      self.dev.dtype_code(self.prev.dtype), self.m, self.n, float(vx), float(vy),
                      self.scratch.data_ptr(), self.record.data_ptr(), self.dev.stream_ptr())
        f, count, flags = self.record.cpu().tolist()
        return f, int(count), int(flags)


@pytest.mark.parametrize("name", CASES)
def test_field_is_the_reference_field(name):
    from pysteps_b200.motion import get_method
    g = np.load(GOLDEN)
    R = build_case(name)
    m, n = R.shape[1:]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = get_method("constant")(R)
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and got.shape == (2, m, n)
    if name in ORDER_DECIDED:
        # the path is decided at a tie of the reference (constant_cases.py): the device ends where the
        # oracle, whose every evaluation it equals bit for bit, ends
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = ora.constant(R)
        assert np.array_equal(_bits(got), _bits(want))
    else:
        assert np.array_equal(_bits(got), _bits(_field(g[name + "/x"], m, n)))


@pytest.mark.parametrize("name", CASES)
def test_every_recorded_evaluation_replayed_on_the_device(name):
    g = np.load(GOLDEN)
    R = np.ma.getdata(build_case(name))
    ev = _Evaluator(R[-2], R[-1])
    for k, (v, want) in enumerate(zip(g[name + "/v"], g[name + "/f"])):
        got = ev(v[0], v[1])
        oracle = ora.evaluate(R[-2], R[-1], v[0], v[1])
        assert got[1:] == oracle[1:] and _same(got[0], oracle[0]), (k, v, got, oracle)
        assert (np.isnan(got[0]) and np.isnan(want)) or abs(got[0] - want) <= 1e-12, (k, v, got[0], want)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_near_half_integer_components_at_large_rows(dtype):
    rng = np.random.default_rng(5)
    m, n = 6000, 5
    R = (rng.standard_normal((2, m, n)) * 4.0).astype(dtype)
    R[0, ::97, 2] = np.nan
    ev = _Evaluator(R[0], R[1])
    comps = (0.5, 0.49999999999999994, -0.5, 2.5, -0.49999999999999994, 1.5000000000000002)
    for vx in comps:
        for vy in comps:
            got = ev(vx, vy)
            want = ora.evaluate(R[0], R[1], vx, vy)
            assert got[1:] == want[1:] and _same(got[0], want[0]), (vx, vy, got, want)


@pytest.mark.parametrize("name", ["shift_256_f64", "shift_256_f32", "nan_blocks_edges_200x180", "one_by_one"])
def test_device_tensor_input_returns_a_device_tensor(name):
    import torch
    from pysteps_b200.motion import get_method
    R = build_case(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = get_method("constant")(R)
        got = get_method("constant")(torch.from_numpy(R).cuda())
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.dtype == torch.float64
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(want))


def test_warnings_follow_the_record():
    """all-NaN overlap: the reference's five RuntimeWarnings of np.mean / np.cov, in order"""
    from pysteps_b200.motion.constant import constant
    R = build_case("all_nan_32x32")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        constant(R)
    first = [str(x.message) for x in w[:5]]
    assert first == ["Mean of empty slice.", "invalid value encountered in divide",
                     "Degrees of freedom <= 0 for slice", "divide by zero encountered in divide",
                     "invalid value encountered in multiply"]
    assert len(w) == 5 * 400
