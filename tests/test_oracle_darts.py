"""CPU: the DARTS oracle (oracle/darts.py, the NumPy restatement of csrc/darts.cu on the same twiddle
tables) against the reference's recorded runs (tests/golden/darts_golden.npz), at the bars of
darts_cases.py: the field, MM, M^H y, and the exception of the MaskedArray case."""
import os

import numpy as np
import pytest

from darts_cases import (CASES, RAISES, build_case, field_bar, field_error, golden_matrix, matrix_bar,
                         matrix_error)
from oracle import darts as ora

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "darts_golden.npz")


@pytest.mark.parametrize("name", [c for c in CASES if c not in RAISES])
def test_oracle_meets_the_bars(name):
    g = np.load(GOLDEN)
    R, kw = build_case(name)
    got, inter = ora.DARTS(R, **kw)
    d, s = field_error(name, got, g, R, kw)
    assert d <= field_bar(name) * s, (d, s)
    for key in ("MM", "Mhy"):
        d, s = matrix_error(inter[key], golden_matrix(g, name, key))
        assert d <= matrix_bar(name) * s, (key, d, s)
    assert g[name + "/margin"] > 1e-8 or (np.isnan(g[name + "/margin"]) and not np.any(g[name + "/MM_upper"]))


def test_masked_nan_raises_the_reference_exception():
    g = np.load(GOLDEN)
    R, kw = build_case("masked_nan_128x96")
    with pytest.raises(np.linalg.LinAlgError) as e:
        ora.DARTS(R, **kw)
    assert f"{type(e.value).__name__}: {e.value}" == str(g["masked_nan_128x96/error"])


def test_tables_use_the_integer_reduced_argument():
    from pysteps_b200.motion.darts import twiddles
    L = 2048
    t = twiddles((-3, 5, 1021), L, -1)
    r = (np.array([-3 % L, 5, 1021])[:, None] * np.arange(L)) % L
    assert np.array_equal(t.real, np.cos(-2.0 * np.pi * r / L)) and np.array_equal(t.imag, np.sin(-2.0 * np.pi * r / L))
    assert np.array_equal(twiddles((-3,), L, -1), twiddles((L - 3,), L, -1))


@pytest.mark.parametrize("name", [c for c in CASES if c not in RAISES])
def test_stored_pixels_match_the_field_rebuilt_from_x(name):
    """the golden holds the reference's x and its field at seeded pixels; the field rebuilt from x by
    numpy's ifft2 (the reference's own last step) must give those pixels"""
    from darts_cases import reference_field, sample_pixels
    g = np.load(GOLDEN)
    R, kw = build_case(name)
    if kw.get("output_type", "spatial") != "spatial":
        pytest.skip("spectral output: the golden's x is the result")
    m, n = R.shape[1:]
    f = reference_field(g[name + "/x"], kw, m, n)
    ys, xs = sample_pixels(m, n)
    assert np.abs(f[:, ys, xs] - g[name + "/pixels"]).max() <= 1e-15 * max(np.abs(f).max(), 1e-300)
