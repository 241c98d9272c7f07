"""Generate tests/golden/probability_golden.npz from the REFERENCE,
pysteps/nowcasts/lagrangian_probability.py, for the cases of probability_cases.py:

    <case>/out        the reference's whole (T, m, n) output            (cases up to 128^2)
    <case>/idx        SAMPLES seeded flat pixel indices                 (LARGE cases)
    <case>/samples    (T, SAMPLES) the reference's output at them       (LARGE cases)
    <case>/nan_count  (T,) NaN pixels of every lead                     (LARGE cases)
    <case>/deviation  max |reference - exact| over the whole output

The reference convolves with scipy's FFT in single precision, so it is not the exact ratio of the
neighbourhood counts.  The generator asserts that the exact oracle (oracle/probability.py) is within
1e-6 of it on every case, with the same NaN pattern, and stores the deviation it found.

    python tests/golden/gen_probability_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from _refimport import ref_module  # noqa: E402
from probability_cases import CASES, LARGE, build_case, sample_index  # noqa: E402
from oracle import probability as ora  # noqa: E402

BOUND = 1e-6


def main():
    ref = ref_module("pysteps.nowcasts.lagrangian_probability")
    out = {}
    for name in CASES:
        args, kw = build_case(name)
        want = ref.forecast(*args, **kw)
        exact = ora.forecast(*args, **kw)
        assert want.dtype == exact.dtype == np.float64 and want.shape == exact.shape, name
        nan = np.isnan(want)
        assert np.array_equal(nan, np.isnan(exact)), name
        dev = float(np.abs(want[~nan] - exact[~nan]).max()) if (~nan).any() else 0.0
        assert dev <= BOUND, (name, dev)
        out[name + "/deviation"] = np.float64(dev)
        if name in LARGE:
            idx = sample_index(name, want.shape[1:])
            out[name + "/idx"] = idx.astype(np.int32)
            out[name + "/samples"] = want.reshape(want.shape[0], -1)[:, idx]
            out[name + "/nan_count"] = nan.reshape(want.shape[0], -1).sum(axis=1)
        else:
            out[name + "/out"] = want
        print(f"{name}: {want.shape}, max |reference - exact| = {dev:.3g}")
    path = os.path.join(HERE, "probability_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
