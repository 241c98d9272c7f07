"""Generate tests/golden/detscores_golden.npz from the REFERENCE, pysteps/verification/detcatscores.py,
detcontscores.py, spatialscores.py and ensscores.py, for the calls of tests/detscores_cases.py:golden_calls(), in the
encoding of gen_verification_golden.py:

    keys       the calls, in order; for call i:
    sig[i]     the outcome's types and shapes (dict keys, Python or NumPy scalar types, dtypes) or the
               exception and its message
    vals       the outcomes' values bit for bit, call i at bytes off[i] .. off[i + 1] (uint8)
    warnings[i]  "Category: message" of every warning the call raised, in order, one per line
    next[i]    NaN (these calls draw no random numbers)

The inputs are rebuilt from seeded generators, so only outcomes are stored.  The generator asserts
that the oracle (oracle/detscores.py) is bit-identical to the reference on every accumulation.

    python tests/golden/gen_detscores_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, "tests")]

from detscores_cases import golden_calls, numpy_moments, reference_modules, run_call  # noqa: E402
from oracle import detscores as ora  # noqa: E402
from verification_cases import encode  # noqa: E402


def check_oracle(fn, args, kwargs, out):
    """the oracle's accumulation against the reference's outcome"""
    if isinstance(out, Exception):
        return
    if fn == "det_cat_fct_accum":
        (thr, axis), data = args[0], args[1:]
        want = [np.zeros_like(out["hits"]) for _ in range(4)]
        ax = (axis,) if isinstance(axis, int) else axis
        for pred, obs in data:
            for w, c in zip(want, ora.contab(pred, obs, thr, tuple(range(pred.ndim)) if ax is None else ax)):
                w += c
        for key, w in zip(("hits", "false_alarms", "misses", "correct_negatives"), want):
            assert np.array_equal(out[key], w), key
    elif fn == "det_cont_fct_accum":
        (axis, cond, thr), data = args[0], args[1:]
        for pred, obs in data:
            ax = tuple(range(pred.ndim)) if axis is None else ((axis,) if isinstance(axis, int) else axis)
            check_moments(pred, obs, ax, cond, thr)
    elif fn == "fss_accum":
        (thr, scale), data = args[0], args[1:]
        tot = [0.0, 0.0, 0.0]
        for X_f, X_o in data:
            tot = [t + v for t, v in zip(tot, ora.fss_sums(X_f, X_o, thr, scale))]
        for key, t in zip(("sum_obs_sq", "sum_fct_obs", "sum_fct_sq"), tot):
            assert np.float64(out[key]).tobytes() == np.float64(t).tobytes(), key
    elif fn == "fss":
        X_f, X_o, thr, scale = args
        oo, fo, ff = ora.fss_sums(X_f, X_o, thr, scale)
        with np.errstate(invalid="ignore"):
            assert np.float64(out).tobytes() == np.float64(1.0 - (ff - 2.0 * fo + oo) / (ff + oo)).tobytes()
    elif fn == "ensemble_spread" and args[1] == "fss":
        assert np.float64(out).tobytes() == np.mean(ora.spread_fss(args[0], kwargs["thr"], kwargs["scale"])).tobytes()


def check_moments(pred, obs, axis, cond, thr):
    """the oracle's sums of det_cont_fct_accum, divided as NumPy divides, against np.nanmean"""
    tot, cnt, n = ora.cont_sums(pred, obs, axis, cond, thr)
    want, want_n = numpy_moments(pred, obs, axis, cond, thr)
    with np.errstate(all="ignore"):
        for t, c, w in zip(tot, cnt, want):
            assert (t.astype(np.float64) / c).astype(w.dtype).tobytes() == np.asarray(w).tobytes()
    assert np.array_equal(n, want_n)


def main():
    ref = reference_modules()
    assert ref is not None, "the reference is not importable"
    keys, sigs, vals, off, warns = [], [], [], [0], []
    for key, mod, fn, args, kwargs in golden_calls():
        out, warned = run_call(ref[mod], fn, args, kwargs)
        check_oracle(fn, args, kwargs, out)
        sig, v = encode(out)
        keys.append(key)
        sigs.append(sig)
        vals.append(v)
        off.append(off[-1] + len(v))
        warns.append("\n".join(warned))
    assert len(set(keys)) == len(keys)
    store = dict(keys=np.array(keys), sig=np.array(sigs), vals=np.concatenate(vals), off=np.array(off, np.int64),
                 warnings=np.array(warns), next=np.full(len(keys), np.nan))
    path = os.path.join(HERE, "detscores_golden.npz")
    np.savez_compressed(path, **store)
    print(f"{path}: {len(keys)} calls, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
