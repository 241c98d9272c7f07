"""GPU: the DARTS method (csrc/darts.cu behind motion/darts.py) against the reference's recorded runs
(tests/golden/darts_golden.npz) at the bars of darts_cases.py, intermediates included; repeated
calls bit-identical; CUDA-tensor input, float32 tensors and spectral output on the device."""
import os

import numpy as np
import pytest

from darts_cases import (CASES, RAISES, build_case, field_bar, field_error, golden_matrix, matrix_bar,
                         matrix_error)

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "darts_golden.npz")


def _device_normal(R, kw):
    """(spectrum, MM, M^H y) from the device entry points, read back"""
    import torch
    from pysteps_b200 import _device, _lib
    from pysteps_b200.motion import darts as d
    _device.require_cuda()
    N_x, N_y, N_t, M_x, M_y = (kw.get(k, v) for k, v in (("N_x", 50), ("N_y", 50), ("N_t", 4), ("M_x", 2), ("M_y", 2)))
    T, m, n = R.shape
    frames = _device.to_device(np.ascontiguousarray(np.ma.getdata(R)))
    tw_x, tw_y, tw_t, K = d.spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y)
    Kt, Ky, Kx = tw_t.shape[0], tw_y.shape[0], 2 * K + 1
    tabs = [_device.to_device(np.ascontiguousarray(t)) for t in (tw_x, tw_y, tw_t)]
    work = torch.empty(T * m * tw_x.shape[0] + Kt * m * Kx, dtype=torch.complex128, device="cuda")
    spec = torch.empty((Kt, Ky, Kx), dtype=torch.complex128, device="cuda")
    s = _device.stream_ptr()
    _lib.call("b200_darts_spectrum", frames.data_ptr(), _device.dtype_code(frames.dtype), T, m, n, tabs[0].data_ptr(),
              tw_x.shape[0], tabs[1].data_ptr(), Ky, tabs[2].data_ptr(), Kt, K, work.data_ptr(), spec.data_ptr(), s)
    nc = 2 * (2 * M_x + 1) * (2 * M_y + 1)
    rows = Kt * (2 * N_y + 1) * (2 * N_x + 1)
    part = torch.empty(-(-rows // d.NORMAL_ROWS) * (nc * (nc + 1) // 2 + nc), dtype=torch.complex128, device="cuda")
    out = torch.empty(nc * (nc + 1), dtype=torch.complex128, device="cuda")
    c1 = -1.0 * T / (n * m)
    _lib.call("b200_darts_normal", spec.data_ptr(), N_x, N_y, N_t, M_x, M_y, c1 / n, c1 / m, part.data_ptr(),
              out.data_ptr(), out[nc * nc:].data_ptr(), s)
    o = out.cpu().numpy()
    return spec.cpu().numpy(), o[: nc * nc].reshape(nc, nc), o[nc * nc:]


@pytest.mark.parametrize("name", [c for c in CASES if c not in RAISES])
def test_field_and_intermediates_meet_the_bars(name):
    from oracle import darts as ora
    from pysteps_b200.motion import get_method
    g = np.load(GOLDEN)
    R, kw = build_case(name)
    got = get_method("darts")(R, **kw)
    assert isinstance(got, np.ndarray)
    d, s = field_error(name, got, g, R, kw)
    print(f"{name}: field max|d| / max|field| = {d / s if s else d:.3e}")
    assert d <= field_bar(name) * s, (d, s)
    spec, MM, Mhy = _device_normal(R, kw)
    for key, a in (("MM", MM), ("Mhy", Mhy)):
        d, s = matrix_error(a, golden_matrix(g, name, key))
        print(f"{name}: {key} max|d| / max = {d / s if s else d:.3e}")
        assert d <= matrix_bar(name) * s, (key, d, s)
    if R.size <= 1 << 20:  # the spectrum block against the oracle's direct DFT on the same tables
        want = ora.spectrum(np.ma.getdata(R), **{k: v for k, v in kw.items() if k[0] in "NM"})
        assert np.abs(spec - want).max() <= 1e-12 * max(np.abs(want).max(), 1.0)


def test_masked_nan_raises_the_reference_exception():
    from pysteps_b200.motion import get_method
    g = np.load(GOLDEN)
    R, kw = build_case("masked_nan_128x96")
    with pytest.raises(np.linalg.LinAlgError) as e:
        get_method("darts")(R, **kw)
    assert f"{type(e.value).__name__}: {e.value}" == str(g["masked_nan_128x96/error"])


@pytest.mark.parametrize("name", ["shift_256_f64", "alias_80x90", "lsq1_128x128"])
def test_repeated_calls_are_bit_identical(name):
    from pysteps_b200.motion import get_method
    R, kw = build_case(name)
    a = get_method("darts")(R, **kw)
    b = get_method("darts")(R, **kw)
    assert np.array_equal(a.view(np.int64), b.view(np.int64))
    sa, sb = _device_normal(R, kw), _device_normal(R, kw)
    for x, y in zip(sa, sb):
        assert np.array_equal(x.view(np.int64), y.view(np.int64))


@pytest.mark.parametrize("name", ["shift_256_f64", "shift_256_f32", "odd_97x131", "spectral_128x112"])
def test_device_tensor_input_returns_the_numpy_result_on_the_device(name):
    import torch
    from pysteps_b200.motion import get_method
    g = np.load(GOLDEN)
    R, kw = build_case(name)
    want = get_method("darts")(R, **kw)
    got = get_method("darts")(torch.from_numpy(R).cuda(), **kw)
    assert isinstance(got, torch.Tensor) and got.is_cuda
    assert got.dtype == (torch.complex128 if kw.get("output_type") == "spectral" else torch.float64)
    got = got.cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got.view(np.int64), want.view(np.int64))
    d, s = field_error(name, got, g, R, kw)
    assert d <= field_bar(name) * s, (d, s)
