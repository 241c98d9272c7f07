"""Generate tests/golden/darts_golden.npz from the REFERENCE, pysteps/motion/darts.py, for the cases of
darts_cases.py.  The reference's solve is wrapped to record its own matrices:

    <case>/x        the solution (n_c); the result is darts_cases.reference_field(x), asserted bit for bit
    <case>/pixels   the spatial field (2, count) at darts_cases.sample_pixels
    <case>/MM_upper the upper triangle of M^H M, row by row, and <case>/Mhy M^H y (n_c), from the
                    reference's M and y
    <case>/s        the singular values of MM
    <case>/margin   min_i |s_i - cut| / s_0, cut = 0.01 s_0 (lsq_method 2) or 1e-4 s_0 (lsq_method 1);
                    asserted > 1e-8 so that no case sits on the cut (NaN for a zero MM)
    <case>/error    for a case that raises: "<type>: <message>"

    python tests/golden/gen_darts_golden.py
"""
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from _refimport import ref_module  # noqa: E402
from darts_cases import CASES, build_case, reference_field, sample_pixels  # noqa: E402


def _record_gram(rec, M, y, cut):
    M_ct = M.conjugate().T
    MM = np.dot(M_ct, M)
    rec["MM_upper"], rec["Mhy"] = MM[np.triu_indices(MM.shape[0])], np.dot(M_ct, y)
    s = np.linalg.svd(MM, compute_uv=False)
    rec["s"] = s
    rec["margin"] = np.min(np.abs(s - cut * s[0])) / s[0] if s[0] > 0 else np.nan


def record(R, kw):
    ref = ref_module("pysteps.motion.darts")
    rec = {}
    real_leastsq, real_lstsq = ref._leastsq, ref.lstsq

    def leastsq(A, B, y):
        _record_gram(rec, np.hstack([A, B]), y, 0.01)
        rec["x"] = real_leastsq(A, B, y)
        return rec["x"]

    def lstsq(M, y, rcond=None):
        _record_gram(rec, M, y, 1e-4)
        out = real_lstsq(M, y, rcond=rcond)
        rec["x"] = out[0]
        return out

    with mock.patch.object(ref, "_leastsq", leastsq), mock.patch.object(ref, "lstsq", lstsq):
        try:
            rec["field"] = ref.DARTS(R, **kw)
        except Exception as e:  # noqa: BLE001 -- the exception is the result
            rec["error"] = np.array(f"{type(e).__name__}: {e}")
    return rec


def main():
    out = {}
    for name in CASES:
        R, kw = build_case(name)
        rec = record(R, kw)
        if "field" in rec:
            f = rec.pop("field")
            m, n = R.shape[1:]
            rebuilt = reference_field(rec["x"], kw, m, n)
            assert rebuilt.dtype == f.dtype and np.array_equal(rebuilt.view(np.int64), f.view(np.int64)), name
            if kw.get("output_type", "spatial") == "spatial":
                ys, xs = sample_pixels(m, n)
                rec["pixels"] = f[:, ys, xs]
        if "margin" in rec and np.isfinite(rec["margin"]):
            assert rec["margin"] > 1e-8, (name, rec["margin"])
        for k, v in rec.items():
            out[name + "/" + k] = v
        print(f"{name}: margin {rec.get('margin')}, error {rec.get('error')}")
    path = os.path.join(HERE, "darts_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
