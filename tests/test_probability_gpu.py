"""GPU: the local Lagrangian probability nowcast (csrc/probability.cu behind
nowcasts/lagrangian_probability.py) against the exact oracle (oracle/probability.py), bit for bit,
and against the reference's stored outputs (tests/golden/probability_golden.npz), within 1e-6."""
import os

import numpy as np
import pytest

from conftest import assert_bits_equal
from oracle import probability as ora
from probability_cases import CASES, LARGE, build_case, sample_index
from pysteps_b200 import _synthetic as syn

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "probability_golden.npz")
BOUND = 1e-6


def _forecast():
    import pysteps_b200
    return pysteps_b200.nowcasts.get_method("probability")


def _close(got, want, what):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    if (~nan).any():
        assert np.abs(got[~nan] - want[~nan]).max() <= BOUND, what


@pytest.mark.parametrize("name", CASES)
def test_golden_case(name):
    args, kw = build_case(name)
    got = _forecast()(*args, **kw)
    assert_bits_equal(got, ora.forecast(*args, **kw), name)
    g = np.load(GOLDEN)
    if name in LARGE:
        idx = sample_index(name, got.shape[1:])
        _close(got.reshape(got.shape[0], -1)[:, idx], g[name + "/samples"], name)
        assert np.array_equal(np.isnan(got).reshape(got.shape[0], -1).sum(axis=1), g[name + "/nan_count"])
    else:
        _close(got, g[name + "/out"], name)


def test_2048_t12_and_device_tensors():
    import torch
    P = syn.nan_disc(syn.rain_field(2048, 2048, 21), 0.1)
    V = syn.velocity_field(2048, 2048, 21)
    fc = _forecast()
    got = fc(P, V, 12, 5.0)
    assert_bits_equal(got, ora.forecast(P, V, 12, 5.0), "2048^2 T=12")
    dev = fc(torch.from_numpy(P).cuda(), torch.from_numpy(V).cuda(), 12, 5.0)
    assert dev.is_cuda and dev.dtype == torch.float64
    assert_bits_equal(dev.cpu().numpy(), got, "CUDA-tensor call")
    assert_bits_equal(fc(P, V, 12, 5.0), got, "repeated call")


def test_float32_device_tensors_and_list_timesteps():
    import torch
    P = syn.nan_disc(syn.rain_field(200, 150, 22)).astype(np.float32)
    V = syn.velocity_field(200, 150, 22)
    T = [0.1, 1.0, 2.5, 7.0]
    got = _forecast()(P, V, T, 5.0, slope=4.5)
    dev = _forecast()(torch.from_numpy(P).cuda(), torch.from_numpy(V).cuda(), T, 5.0, slope=4.5)
    assert_bits_equal(dev.cpu().numpy(), got, "float32 CUDA-tensor call")
    assert_bits_equal(got, ora.forecast(P, V, T, 5.0, slope=4.5), "float32 list")


def test_all_nan_lead_gives_an_all_nan_plane():
    # a uniform flow of 40 px per step takes every pixel of a 32 px wide frame from outside, where
    # outval is NaN
    P = syn.rain_field(24, 32, 23)
    V = np.stack([np.full((24, 32), 40.0), np.zeros((24, 32))])
    got = _forecast()(P, V, 3, 5.0)
    assert np.isnan(got).all()
    assert_bits_equal(got, ora.forecast(P, V, 3, 5.0), "all-NaN leads")


@pytest.mark.parametrize("shape", [(1, 97), (83, 1), (1, 1)])
def test_single_row_and_column_frames(shape):
    P = np.arange(np.prod(shape), dtype=np.float64).reshape(shape) % 7
    if P.size > 1:
        P[tuple(k // 2 for k in shape)] = np.nan
    V = np.zeros((2,) + shape)
    for method in ("semilagrangian", "eulerian"):
        got = _forecast()(P, V, 5, 3.0, extrap_method=method, slope=3)
        assert_bits_equal(got, ora.forecast(P, V, 5, 3.0, extrap_method=method, slope=3), f"{shape} {method}")
