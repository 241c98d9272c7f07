"""Generate tests/golden/probmatching_golden.npz from the REFERENCE,
pysteps/postprocessing/probmatching.py, for the cases of probmatching_cases.py:

    <case>/out        the reference's whole output                               (small cases)
    <case>/idx        SAMPLES seeded flat pixel indices                          (LARGE cases)
    <case>/samples    the reference's output at them                             (LARGE cases)
    <case>/sha        SHA-256 of the output's sorted bit patterns (its values)   (LARGE cases)
    <case>/stable     the output with ties in pixel order (TIES cases; sampled for LARGE ones)
    <case>/error      "Type: message" of the exception a call raises             (ERRORS cases)
    <case>/warnings   "Category: message" of every warning the call raised, in order
    <case>/next       np.random.random() (or the case's RandomState's random()) right after the call

The generator asserts that the oracle (oracle/probmatching.py) is bit-identical to the reference on
every case without ties, and equal within every tie group on the TIES cases.

    python tests/golden/gen_probmatching_golden.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from _refimport import ref_module  # noqa: E402
from oracle import probmatching as ora  # noqa: E402
from probmatching_cases import (CASES, ERRORS, LARGE, TIES, build_case, multiset_sha, sample_index,  # noqa: E402
                                seed_of, tie_equal)


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    it = {4: np.int32, 8: np.int64}[a.dtype.itemsize]
    return np.array_equal(na, nb) and np.array_equal(a.view(it)[~na], b.view(it)[~nb])


def run_case(ref, name):
    """(output or exception, warnings, next draw, draws) of the reference on case `name`"""
    fn, args, kw = build_case(name)
    rs = kw.get("randgen")
    if rs is None:
        np.random.seed(seed_of(name))
    gen = rs if rs is not None else np.random
    state = gen.get_state()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            out = (ref.nonparam_match_empirical_cdf if fn == "match" else ref.resample_distributions)(*args, **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            out = e
    nxt = gen.random()
    draws = None
    if fn == "resample" and not isinstance(out, Exception):
        gen.set_state(state)
        draws = gen.binomial(1, np.clip(args[2], 0.0, 1.0), np.asarray(args[0]).size)
    return out, [f"{x.category.__name__}: {x.message}" for x in w], nxt, draws


def main():
    ref = ref_module("pysteps.postprocessing.probmatching")
    out = {}
    for name in CASES:
        fn, args, kw = build_case(name)
        want, warned, nxt, draws = run_case(ref, name)
        out[name + "/warnings"] = np.array(warned, dtype=str)
        out[name + "/next"] = np.float64(nxt)
        if name in ERRORS:
            assert isinstance(want, Exception), name
            out[name + "/error"] = np.array(f"{type(want).__name__}: {want}")
            print(f"{name}: {type(want).__name__}: {want}")
            continue
        assert not isinstance(want, Exception), (name, want)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            if fn == "match":
                exact = ora.nonparam_match_empirical_cdf(*args, **kw)
            else:
                exact = ora.resample_distributions(args[0], args[1], draws)
        if name in TIES:
            assert tie_equal(exact, want, args[0], kw.get("ignore_indices")), name
        else:
            assert bits_equal(want, exact), name
        if name in LARGE:
            idx = sample_index(name, want.size)
            out[name + "/idx"] = idx.astype(np.int32)
            out[name + "/samples"] = want.reshape(-1)[idx]
            out[name + "/sha"] = np.array(multiset_sha(want))
            if name in TIES:
                out[name + "/stable"] = exact.reshape(-1)[idx]
        else:
            out[name + "/out"] = want
            if name in TIES:
                out[name + "/stable"] = exact
        print(f"{name}: {want.dtype} {want.shape}, warnings {warned}, "
              f"{'ties differ' if name in TIES and not bits_equal(want, exact) else 'exact'}")
    path = os.path.join(HERE, "probmatching_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
