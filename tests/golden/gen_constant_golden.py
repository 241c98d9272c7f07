"""Generate tests/golden/constant_golden.npz from the REFERENCE, pysteps/motion/constant.py, for the
cases of constant_cases.py.  For every case it stores the reference's result.x and the whole
sequence of points v and objective values f(v) that scipy's Nelder-Mead asked for, recorded by
wrapping the objective that op.minimize receives:

    <case>/x      result.x (2,)
    <case>/v      (K, 2) the evaluated points, in order
    <case>/f      (K,)   the reference's f at each of them

    python tests/golden/gen_constant_golden.py
"""
import os
import sys
import warnings
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from _refimport import ref_module  # noqa: E402
from constant_cases import CASES, build_case  # noqa: E402


def record(R):
    """Run the reference on R -> (result.x, points, values)."""
    ref = ref_module("pysteps.motion.constant")
    real = ref.op.minimize
    seen = []
    out = {}

    def minimize(fun, x0, **kw):
        def wrapped(v):
            f = fun(v)
            seen.append((np.array(v, dtype=np.float64), float(f)))
            return f
        res = real(wrapped, x0, **kw)
        out["x"] = np.array(res.x, dtype=np.float64)
        return res

    with mock.patch.object(ref.op, "minimize", minimize), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        field = ref.constant(R)
    m, n = R.shape[1:]
    assert np.array_equal(field, np.stack([-out["x"][0] * np.ones((m, n)), -out["x"][1] * np.ones((m, n))]))
    return out["x"], np.array([v for v, _ in seen]).reshape(-1, 2), np.array([f for _, f in seen])


def main():
    out = {}
    for name in CASES:
        x, v, f = record(build_case(name))
        out[name + "/x"], out[name + "/v"], out[name + "/f"] = x, v, f
        print(f"{name}: {len(f)} evaluations, x = {x.tolist()}")
    path = os.path.join(HERE, "constant_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
