"""Inputs of the local Lagrangian probability goldens (tests/golden/probability_golden.npz), shared by
the generator, the CPU tests and the GPU tests.  build_case(name) -> (args, kwargs) of
``forecast(precip, velocity, timesteps, threshold, **kwargs)``.

Cases up to 128^2 store the reference's whole output; LARGE cases store SAMPLES seeded pixels of
every lead and each lead's NaN count."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from pysteps_b200 import _synthetic as syn  # noqa: E402

SAMPLES = 1024
LARGE = ("f64_512_T6", "f64_1024_T12")


def _rain(m, n, seed, dtype=np.float64):
    return syn.rain_field(m, n, seed).astype(dtype)


def _vel(m, n, seed, kind="smooth"):
    return syn.velocity_field(m, n, seed, kind)


def _f32_threshold_field():
    """float32 rain whose wet pixels are exactly float32(0.1): with the threshold float(float32(0.1)) +
    1e-12 they exceed, because NumPy compares a float32 field with a Python float in float32"""
    r = _rain(48, 48, 8)
    return np.where(r > 0, np.float32(0.1), np.float32(0.0)).astype(np.float32)


def _ref_example():
    p = np.zeros((20, 20))
    p[5:10, 5:10] = 1
    return p


def build_case(name):
    c = {
        "f64_128x64_T3": lambda: ((_rain(128, 64, 1), _vel(128, 64, 1), 3, 5.0), {}),
        "f32_64_T3": lambda: ((_rain(64, 64, 2, np.float32), _vel(64, 64, 2), 3, 5.0), {}),
        "nan_96x64": lambda: ((syn.nan_disc(_rain(96, 64, 3), 0.2), _vel(96, 64, 3), 3, 2.0), {}),
        "list_fractional": lambda: ((_rain(48, 56, 4), _vel(48, 56, 4), [0.1, 0.5, 1.5, 2.25], 5.0), {}),
        "slope_float": lambda: ((_rain(48, 48, 5), _vel(48, 48, 5), 3, 5.0), {"slope": 2.7}),
        "slope_zero": lambda: ((syn.nan_disc(_rain(48, 48, 6)), _vel(48, 48, 6), 3, 5.0), {"slope": 0}),
        "kernel_over_frame_48x80": lambda: ((_rain(48, 80, 7), _vel(48, 80, 7), [1, 6, 12], 5.0), {}),
        "odd_width_40x97": lambda: ((syn.nan_disc(_rain(40, 97, 9)), _vel(40, 97, 9), 2, 1.0), {}),
        "f32_threshold_rounding": lambda: ((_f32_threshold_field(), _vel(48, 48, 8), 2,
                                            float(np.float32(0.1)) + 1e-12), {}),
        "f32_nan_counts_3e8": lambda: ((syn.nan_disc(_rain(48, 48, 10, np.float32), 0.25), _vel(48, 48, 10), 2,
                                        3e8), {}),
        "inf_threshold": lambda: ((syn.nan_disc(_rain(48, 48, 11), 0.25), _vel(48, 48, 11), 2, np.inf), {}),
        "eulerian": lambda: ((syn.nan_disc(_rain(48, 80, 12)), _vel(48, 80, 12), 2, 5.0),
                             {"extrap_method": "eulerian"}),
        "extrap_kwargs": lambda: ((_rain(48, 48, 13), _vel(48, 48, 13), 3, 5.0),
                                  {"extrap_kwargs": {"vel_timestep": 2, "interp_order": 3, "outval": 0.0}}),
        "reference_example_20x20": lambda: ((_ref_example(), np.zeros((2, 20, 20)), 4, 0.5), {"slope": 1}),
        "f64_512_T6": lambda: ((_rain(512, 512, 14), _vel(512, 512, 14), 6, 5.0), {}),
        "f64_1024_T12": lambda: ((syn.nan_disc(_rain(1024, 1024, 15)), _vel(1024, 1024, 15), 12, 5.0), {}),
    }
    return c[name]()


CASES = ("f64_128x64_T3", "f32_64_T3", "nan_96x64", "list_fractional", "slope_float", "slope_zero",
         "kernel_over_frame_48x80", "odd_width_40x97", "f32_threshold_rounding", "f32_nan_counts_3e8",
         "inf_threshold", "eulerian", "extrap_kwargs", "reference_example_20x20") + LARGE


def sample_index(name, shape):
    """the seeded flat pixel indices stored for a LARGE case (the same for every lead)"""
    rng = np.random.default_rng(sum(map(ord, name)))
    return np.sort(rng.choice(shape[0] * shape[1], SAMPLES, replace=False))
