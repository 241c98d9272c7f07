"""CPU: the probability-matching oracle (oracle/probmatching.py) against the reference's stored
outputs (tests/golden/probmatching_golden.npz) and, where it is importable, against the live reference:
bit for bit, and on the cases with tied initial values equal within every tie group."""
import os
import warnings

import numpy as np
import pytest

from conftest import assert_bits_equal
from oracle import probmatching as ora
from probmatching_cases import (CASES, ERRORS, LARGE, TIES, build_case, multiset_sha, rain, sample_index, seed_of,
                                tie_equal)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "probmatching_golden.npz")
_golden = {}


def golden():
    """the stored arrays, read once (the file is closed, so no ResourceWarning reaches a recorded call)"""
    if not _golden:
        with np.load(GOLDEN) as g:
            _golden.update({k: g[k] for k in g.files})
    return _golden


def draws_of(name):
    """the 0/1 draws the reference takes in resample case `name`, from the case's random state"""
    fn, args, kw = build_case(name)
    gen = kw.get("randgen")
    if gen is None:
        np.random.seed(seed_of(name))
        gen = np.random
    return gen.binomial(1, np.clip(args[2], 0.0, 1.0), np.asarray(args[0]).size)


def oracle_call(name):
    fn, args, kw = build_case(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if fn == "match":
            return ora.nonparam_match_empirical_cdf(*args, **kw)
        return ora.resample_distributions(args[0], args[1], draws_of(name))


def check_golden(name, got, stable=True):
    """got (the full output of case `name`) against the stored outputs: the stable-order output bit for
    bit on TIES cases (stable=True), the reference's elsewhere; LARGE cases at their samples and as a
    multiset"""
    g = golden()
    fn, args, kw = build_case(name)
    if name in LARGE:
        flat = np.asarray(got).reshape(-1)
        idx = sample_index(name, flat.size)
        assert np.array_equal(g[name + "/idx"], idx)
        want = g[name + "/stable"] if name in TIES and stable else g[name + "/samples"]
        if name in TIES and not stable:
            return
        assert_bits_equal(flat[idx], want, name)
        assert multiset_sha(got) == str(g[name + "/sha"]), name
    elif name in TIES:
        if stable:
            assert_bits_equal(got, g[name + "/stable"], name)
        assert tie_equal(got, g[name + "/out"], args[0], kw.get("ignore_indices")), name
    else:
        assert_bits_equal(got, g[name + "/out"], name)


@pytest.mark.parametrize("name", [c for c in CASES if c not in ERRORS])
def test_oracle_matches_the_golden(name):
    check_golden(name, oracle_call(name))


def _reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module("pysteps.postprocessing.probmatching")


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_the_live_reference_on_random_fields(seed):
    ref = _reference()
    rng = np.random.default_rng(300 + seed)
    for _ in range(20):
        shape = (int(rng.integers(1, 40)), int(rng.integers(1, 40)))
        x = rain(shape, int(rng.integers(1 << 30)), dry=float(rng.random()))
        t = rain(shape, int(rng.integers(1 << 30)), dry=float(rng.random()))
        if rng.random() < 0.3:
            t[rng.random(shape) < 0.1] = np.nan
        kw = {}
        if rng.random() < 0.3:
            x[rng.random(shape) < 0.1] = np.nan
            kw["ignore_indices"] = np.isnan(x)
        if np.isnan(x).all():
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = ref.nonparam_match_empirical_cdf(x, t, **kw)
            got = ora.nonparam_match_empirical_cdf(x, t, **kw)
        assert tie_equal(got, want, x, kw.get("ignore_indices"))
        a, b = rain(shape, seed), rain(shape, seed + 1)
        np.random.seed(seed)
        want = ref.resample_distributions(a, b, 0.3)
        np.random.seed(seed)
        got = ora.resample_distributions(a, b, np.random.binomial(1, 0.3, a.size))
        assert_bits_equal(got, want)


def test_percentile_taps_are_numpys():
    """_lerp at the oracle's taps equals np.percentile for every wet count of small arrays"""
    rng = np.random.default_rng(9)
    for n in (1, 2, 3, 7, 10, 97, 101, 1000):
        s = np.sort(rng.gamma(0.8, 2.0, n))
        for x_wet in range(0, n + 1):
            i0, i1, gamma = ora.percentile_taps(n, x_wet)
            want = np.percentile(s, 100 * (1 - np.int64(x_wet) / n))
            assert ora.lerp(s[i0], s[i1], gamma) == want, (n, x_wet)
