"""Generate tests/golden/verification_golden.npz from the REFERENCE, pysteps/verification/probscores.py
and ensscores.py, for the calls of tests/verification_cases.py:golden_calls():

    keys       the calls, in order; for call i:
    sig[i]     the outcome's types and shapes (tuple, list, dict keys, Python or NumPy scalar types,
               dtypes) or the exception and its message
    vals       the outcomes' values bit for bit, call i at bytes off[i] .. off[i + 1] (uint8)
    warnings[i]  "Category: message" of every warning the call raised, in order, one per line
    next[i]    np.random.random() right after the call (NaN where it is not seeded: the seed is part
               of the call)

The inputs are rebuilt from seeded generators, so only outcomes are stored.  The generator asserts
that the oracle (oracle/verification.py) is bit-identical to the reference on every accumulation.

    python tests/golden/gen_verification_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, "tests")]

from oracle import verification as ora  # noqa: E402
from verification_cases import encode, golden_calls, reference, run_call  # noqa: E402


def check_oracle(fn, args, out, seed):
    """the oracle's accumulation against the reference's dict"""
    if fn == "CRPS_accum":
        s, n = ora.crps(*args[1:])
        assert out["CRPS_sum"].tobytes() == np.float64(0.0 + s).tobytes() and out["n"] == n
    elif fn == "rankhist_accum":
        (k, xm), X_f, X_o = args
        pairs = ora.rankhist(X_f, X_o, xm)[1]
        np.random.seed(seed)
        u = np.random.uniform(size=len(pairs)) if len(pairs) else np.zeros(0)
        assert np.array_equal(out["n"], ora.rankhist(X_f, X_o, xm, u))
    elif fn == "reldiag_accum":
        (xm, nb, mc), P, O = args
        count, above, sums = ora.reldiag(P, O, xm, out["bin_edges"])
        keep = count >= mc
        assert np.array_equal(out["num_idx"], np.where(keep, count, 0))
        assert np.array_equal(out["Y_sum"], np.where(keep, above, 0))
        assert out["X_sum"].tobytes() == np.where(keep, sums.astype(np.float64), 0.0).tobytes()
    elif fn == "ROC_curve_accum":
        (xm, nb), P, O = args
        for key, v in zip(("hits", "misses", "false_alarms", "corr_neg"), ora.roc(P, O, xm, out["prob_thrs"])):
            assert np.array_equal(out[key], v), key


def main():
    ref = reference()
    assert ref is not None, "the reference is not importable"
    mods = {"probscores": ref[0], "ensscores": ref[1]}
    keys, sigs, vals, off, warns, nexts = [], [], [], [0], [], []
    for key, mod, fn, args, seed in golden_calls():
        out, warned, nxt = run_call(mods[mod], fn, args, seed)
        assert not isinstance(out, Exception), (key, out)
        check_oracle(fn, args, out, seed)
        sig, v = encode(out)
        keys.append(key)
        sigs.append(sig)
        vals.append(v)
        off.append(off[-1] + len(v))
        warns.append("\n".join(warned))
        nexts.append(nxt if seed is not None else np.nan)
    store = dict(keys=np.array(keys), sig=np.array(sigs), vals=np.concatenate(vals), off=np.array(off, np.int64),
                 warnings=np.array(warns), next=np.array(nexts))
    path = os.path.join(HERE, "verification_golden.npz")
    np.savez_compressed(path, **store)
    print(f"{path}: {len(golden_calls())} calls, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
