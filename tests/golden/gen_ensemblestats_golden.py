"""Generate tests/golden/ensemblestats_golden.npz from the REFERENCE,
pysteps/postprocessing/ensemblestats.py, for the cases of ensemblestats_cases.py:

    <case>/out        the reference's whole output                        (small cases)
    <case>/idx        SAMPLES seeded flat pixel indices                   (LARGE cases)
    <case>/samples    (planes, SAMPLES) the reference's output at them    (LARGE cases)
    <case>/nan_count  (planes,) NaN pixels of every output plane          (LARGE cases)
    <case>/warnings   "Category: message" of every warning the call raised, in order
    <case>/seed       np.random.seed before a banddepth call
    <case>/next       np.random.random() right after that call

The generator asserts that the oracle (oracle/ensemblestats.py) is bit-identical to the reference on
every case: C-order inputs, so NumPy sums over the member axis sequentially.

    python tests/golden/gen_ensemblestats_golden.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from _refimport import ref_module  # noqa: E402
from ensemblestats_cases import CASES, LARGE, build_case, sample_index, seed_of  # noqa: E402
from oracle import ensemblestats as ora  # noqa: E402


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    it = {4: np.int32, 8: np.int64}[a.dtype.itemsize]
    return np.array_equal(na, nb) and np.array_equal(a.view(it)[~na], b.view(it)[~nb])


def run_recording(fn, *args, **kw):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = fn(*args, **kw)
    return out, [f"{x.category.__name__}: {x.message}" for x in w]


def oracle_banddepth(X, seed, **kw):
    """the oracle with the tie-breaks the reference draws after np.random.seed(seed)"""
    thr = kw.get("thr")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if thr is None:
            thr = np.nanmin(X)
        mask, _ = ora.band_mask(X, thr)
        np.random.seed(seed)
        b = np.random.random((X.shape[0], int(mask.sum())))
        return ora.banddepth(X, b, thr=thr, norm=kw.get("norm", False))


def main():
    ref = ref_module("pysteps.postprocessing.ensemblestats")
    out = {}
    for name in CASES:
        fn, args, kw = build_case(name)
        if fn == "banddepth":
            np.random.seed(seed_of(name))
            want, warned = run_recording(ref.banddepth, *args, **kw)
            out[name + "/seed"] = np.int64(seed_of(name))
            out[name + "/next"] = np.float64(np.random.random())
            exact = oracle_banddepth(args[0], seed_of(name), **kw)
        else:
            want, warned = run_recording(getattr(ref, fn), *args, **kw)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                exact = getattr(ora, fn)(*args, **kw)
        assert bits_equal(want, exact), name
        out[name + "/warnings"] = np.array(warned, dtype=str)
        if name in LARGE:
            planes = want.reshape(-1, want.shape[-2] * want.shape[-1])
            idx = sample_index(name, planes.shape[1])
            out[name + "/idx"] = idx.astype(np.int32)
            out[name + "/samples"] = planes[:, idx]
            out[name + "/nan_count"] = np.isnan(planes).sum(axis=1)
        else:
            out[name + "/out"] = want
        print(f"{name}: {want.dtype} {want.shape}, warnings {warned}")
    path = os.path.join(HERE, "ensemblestats_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
