"""The reference goldens of tests/golden/blending_golden.npz: through the host logic on the CPU (entry
points emulated, tests/cpu_abi_blending.py) and through the device (marked gpu).  Exact conversions
are compared bit for bit; "dB" and "dBZ" inputs within the conversion's bound (DESIGN.md section 4)."""
import os

import numpy as np
import pytest
import torch

import cpu_abi_blending
from blending_cases import CASES, EXACT, LARGE, UNSUPPORTED, build_case
from conftest import bits_equal
from gen_blending_golden import reduce_large

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "blending_golden.npz")


def _run(name):
    from pysteps_b200.blending import linear_blending
    args, kw = build_case(name)
    try:
        with np.errstate(all="ignore"):
            out = linear_blending.forecast(*args, **kw)
    except Exception as e:  # noqa: BLE001 -- the exception is the result
        return e
    return out.cpu().numpy() if isinstance(out, torch.Tensor) else out


def check(name, got, exact):
    g = np.load(GOLDEN)
    if name in UNSUPPORTED and isinstance(got, NotImplementedError):
        return
    if name + "/error" in g.files:
        assert isinstance(got, Exception) and f"{type(got).__name__}: {got}" == str(g[name + "/error"]), got
        return
    assert not isinstance(got, Exception), got
    if name in LARGE:
        sample, nan_count = reduce_large(got)
        assert tuple(got.shape) == tuple(g[name + "/shape"]) and nan_count == g[name + "/nan_count"]
        want, got = g[name + "/sample"], sample
    else:
        want = g[name + "/out"]
    if exact:
        assert bits_equal(got, want)
    else:
        assert got.dtype == want.dtype and got.shape == want.shape
        assert np.array_equal(np.isnan(got), np.isnan(want))
        assert np.allclose(got, want, rtol=64 * np.finfo(want.dtype).eps, atol=0, equal_nan=True)


def test_golden_has_the_nan_diff_lead():
    g = np.load(GOLDEN)
    out = g["nan_diff/out"]
    assert np.isnan(out[:, 2]).all() and not np.isnan(out[:, 0]).any()


@pytest.mark.parametrize("name", [c for c in CASES if c not in LARGE])
def test_golden_through_the_host(name):
    with cpu_abi_blending.emulated():
        got = _run(name)
    check(name, got, exact=True)  # the emulated conversion is NumPy's own


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_golden_on_the_device(name):
    check(name, _run(name), exact=name in EXACT)
