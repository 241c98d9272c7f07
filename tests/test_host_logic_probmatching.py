"""CPU test of the HOST logic of pysteps_b200.postprocessing.probmatching (argument checks, the order
of the reference's exceptions and warnings, dtypes, the forms of ignore_indices, the percentile taps and
the random stream), with the entry points of csrc/probmatching.cu emulated by the oracle
(tests/cpu_abi_probmatching.py).  Compared with the stored reference outcomes."""
import warnings

import numpy as np
import pytest

import cpu_abi_probmatching
from probmatching_cases import CASES, ERRORS, LARGE, build_case, rain, seed_of
from test_oracle_probmatching import check_golden, golden



def _ours(fn):
    from pysteps_b200.postprocessing import probmatching
    return probmatching.nonparam_match_empirical_cdf if fn == "match" else probmatching.resample_distributions


def outcome(name):
    """(result or exception, ["Category: message", ...], the next random draw) of case `name`"""
    fn, args, kw = build_case(name)
    gen = kw.get("randgen")
    if gen is None:
        np.random.seed(seed_of(name))
        gen = np.random
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            out = _ours(fn)(*args, **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            out = e
    # a ResourceWarning comes from some other test's object collected during the call
    warned = [f"{x.category.__name__}: {x.message}" for x in w if not issubclass(x.category, ResourceWarning)]
    return out, warned, gen.random()


@pytest.mark.parametrize("name", [c for c in CASES if c not in LARGE])
def test_golden_cases_through_the_host(name):
    with cpu_abi_probmatching.emulated():
        got, warned, nxt = outcome(name)
    g = golden()
    if name in ERRORS:
        assert isinstance(got, Exception) and f"{type(got).__name__}: {got}" == str(g[name + "/error"]), got
    else:
        assert isinstance(got, np.ndarray), got
        check_golden(name, got)
    assert warned == list(g[name + "/warnings"]), name
    assert nxt == g[name + "/next"], "the random state after the call differs from the reference's"


@pytest.mark.parametrize("bad", [np.ma.masked_array(np.zeros((3, 3))), np.zeros((3, 3), np.int32),
                                 np.zeros((3, 3), np.float16), [[0.0, 1.0]]])
def test_unsupported_inputs_raise(bad):
    good = np.zeros((3, 3)) if not isinstance(bad, list) else np.zeros((1, 2))
    with cpu_abi_probmatching.emulated():
        for args in ((bad, good), (good, bad)):
            with pytest.raises(NotImplementedError):
                _ours("match")(*args)
            if not isinstance(bad, list):
                with pytest.raises(NotImplementedError):
                    _ours("resample")(*args, 0.5)


def test_error_order():
    """the reference's order: all-NaN initial, then the size, then a bad index, then non-finite values"""
    with cpu_abi_probmatching.emulated():
        with pytest.raises(ValueError, match="only nans"):
            _ours("match")(np.full(3, np.nan), np.zeros(4), ignore_indices=np.array([7]))
        with pytest.raises(ValueError, match="dimension mismatch"):
            _ours("match")(np.array([np.nan, 1.0]), np.zeros(4), ignore_indices=np.array([7]))
        with pytest.raises(IndexError):
            _ours("match")(np.array([np.nan, 1.0]), np.zeros(2), ignore_indices=np.array([7]))
        with pytest.raises(ValueError, match="non-finite"):
            _ours("match")(np.array([np.inf, 1.0, 2.0]), np.zeros(3))


def test_ignore_index_forms_agree():
    x = rain((20, 30), 1)
    t = rain((20, 30), 2, dry=0.2)
    x[2:5] = np.nan
    mask = np.isnan(x)
    with cpu_abi_probmatching.emulated():
        want = _ours("match")(x, t, ignore_indices=mask)
        for ix in (np.nonzero(mask), slice(2, 5), np.arange(2, 5), [2, 3, 4, 4]):
            assert np.array_equal(_ours("match")(x, t, ignore_indices=ix), want, equal_nan=True)


def test_resample_dtypes_and_stream():
    a32, b32 = rain((10, 10), 3, np.float32), rain((10, 10), 4, np.float32)
    with cpu_abi_probmatching.emulated():
        assert _ours("resample")(a32, b32, 0.5).dtype == np.float32
        assert _ours("resample")(a32, b32.astype(np.float64), 0.5).dtype == np.float64
        a = a32.copy()
        a[0, 0] = np.nan
        assert _ours("resample")(a, b32, 0.5).dtype == np.float64
        rs1, rs2 = np.random.RandomState(5), np.random.RandomState(5)
        out = _ours("resample")(a32, b32, 0.5, randgen=rs1)
        rs2.binomial(1, 0.5, a32.size)
        assert rs1.random() == rs2.random() and out.shape == (100,)
        assert _ours("resample")(np.zeros(0), np.zeros(0), 0.5).shape == (0,)
