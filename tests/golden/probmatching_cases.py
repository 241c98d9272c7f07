"""Inputs of the probability-matching goldens (tests/golden/probmatching_golden.npz), shared by the
generator, the CPU tests and the GPU tests.  build_case(name) -> (function name, args, kwargs) of
``nonparam_match_empirical_cdf(initial, target, ...)`` or ``resample_distributions(first, second, p,
...)``; a resample case with a ``randgen`` kwarg gets a fresh np.random.RandomState(seed_of(name)), one
without it runs after np.random.seed(seed_of(name)).

Cases of up to 2^16 values store the reference's whole output; LARGE cases store SAMPLES seeded pixels,
and the SHA-256 of the output's sorted bit patterns (its multiset of values).  TIES cases have tied
wet initial values: they also store the stable-order output (``<case>/stable``)."""
import numpy as np

SAMPLES = 4096
LARGE = ("match_f64_2048_more_target", "match_f32_2048_fewer_target", "match_f32_2048_more_target")
TIES = ("match_ties_small", "match_ties_negative_zero", "match_f32_2048_fewer_target",
        "match_f32_2048_more_target")
ERRORS = ("match_error_all_nan", "match_error_nonfinite", "match_error_size", "match_error_empty",
          "match_error_ignored_minus_inf", "resample_error_shape")


def rain(shape, seed, dtype=np.float64, dry=0.5):
    """rain-like values, `dry` of them exactly 0"""
    rng = np.random.default_rng(seed)
    X = rng.gamma(0.8, 2.0, shape)
    X[rng.random(shape) < dry] = 0.0
    return X.astype(dtype)


def _f(v):
    return np.array(v, dtype=np.float64)


def _gamma_case(n, gamma_kind):
    """target / initial of n values whose percentile index lands as asked: x_wet initial wet values
    give virtual index (n - 1)(1 - x_wet / n)"""
    for x_wet in range(1, n):
        v = (n - 1) * np.true_divide(100 * (1 - np.int64(x_wet) / n), 100.0)
        g = v - np.floor(v)
        if (gamma_kind == "zero" and g == 0 and v < n - 1) or (gamma_kind == "below_half" and 0.4 < g < 0.5):
            break
    rng = np.random.default_rng(n + x_wet)
    initial = np.zeros(n)
    initial[rng.choice(n, x_wet, replace=False)] = rng.permutation(np.arange(1, x_wet + 1)) * 0.5
    target = rng.gamma(0.8, 2.0, n)
    target[rng.random(n) < 0.1] = 0.0
    return initial, target


def _ignored_cases():
    init = rain((40, 50), 7)
    trg = rain((40, 50), 8, dry=0.3)
    init[:3, :] = np.nan
    mask = np.isnan(init)
    idx = np.flatnonzero(mask.reshape(-1))
    return init, trg, mask, idx


def _cases():
    init_i, trg_i, mask_i, idx_i = _ignored_cases()
    tie_init = _f([0, 1, 1, 1, 2, 2, 0, 3, 3, 3, 3, 0])
    tie_trg = _f([0, 5, 4, 3, 2, 9, 8, 7, 6, 1, 0, 0])
    c = {
        # the reference's own unit cases (pysteps/tests/test_postprocessing_probmatching.py), as floats
        "match_unit_ignore_nans_both": lambda: ("match", (_f([np.nan, np.nan, 6, 2, 0, 0, 0, 0, 0, 0]),
                                                          _f([np.nan, np.nan, 9, 5, 4, 0, 0, 0, 0, 0])),
                                                {"ignore_indices": np.isnan(_f([np.nan, np.nan, 6, 2, 0, 0, 0, 0, 0, 0]))}),
        "match_unit_zeroes_initial": lambda: ("match", (np.zeros(10), _f([0, 2, 3, 4, 5, 6, 7, 8, 9, 10])), {}),
        "match_unit_ignore_nans_initial": lambda: ("match", (_f([0, 1, 2, 3, 4] + [np.nan] * 5),
                                                             _f([0, 2, 3, 4, 5, 6, 7, 8, 9, 10])),
                                                   {"ignore_indices": np.array([False] * 5 + [True] * 5)}),
        "match_unit_ignore_nans_target": lambda: ("match", (np.arange(10.0), _f([0, 2, 3, 4] + [np.nan] * 6)),
                                                  {"ignore_indices": np.array([False] * 4 + [True] * 6)}),
        "match_unit_more_zeroes_initial": lambda: ("match", (_f([1, 4, 0, 0, 0, 0, 0, 0, 0, 0]),
                                                             _f([10, 8, 6, 4, 2, 0, 0, 0, 0, 0])),
                                                   {"ignore_indices": np.zeros(10, bool)}),
        "match_unit_more_zeroes_initial_unsrt": lambda: ("match", (_f([1, 4, 0, 0, 0, 0, 0, 0, 0, 0]),
                                                                   _f([6, 4, 2, 0, 0, 0, 0, 0, 10, 8])), {}),
        "match_unit_more_zeroes_target": lambda: ("match", (_f([1, 3, 7, 5, 0, 0, 0, 0, 0, 0]),
                                                            _f([10, 8, 0, 0, 0, 0, 0, 0, 0, 0])), {}),
        "match_unit_2dim": lambda: ("match", (_f([[1, 3, 5], [11, 9, 7]]), _f([[2, 4, 6], [8, 10, 12]])), {}),
        # rain fields
        "match_f64_2048_more_target": lambda: ("match", (rain((2048, 2048), 1, dry=0.55),
                                                         rain((2048, 2048), 2, dry=0.45)), {}),
        "match_f32_2048_fewer_target": lambda: ("match", (rain((2048, 2048), 3, np.float32, dry=0.45),
                                                          rain((2048, 2048), 4, np.float32, dry=0.55)), {}),
        "match_f32_2048_more_target": lambda: ("match", (rain((2048, 2048), 5, np.float32, dry=0.55),
                                                         rain((2048, 2048), 6, np.float32, dry=0.45)), {}),
        "match_f64_f32_mixed": lambda: ("match", (rain((64, 80), 9), rain((64, 80), 10, np.float32, 0.3)), {}),
        "match_f64_300x200": lambda: ("match", (rain((300, 200), 11), rain((300, 200), 12, dry=0.2)), {}),
        # ignore_indices as a mask, an integer index and a tuple
        "match_ignore_mask": lambda: ("match", (init_i, trg_i), {"ignore_indices": mask_i}),
        "match_ignore_int_index": lambda: ("match", (init_i, trg_i), {"ignore_indices": np.arange(3)}),
        "match_ignore_tuple": lambda: ("match", (init_i, trg_i), {"ignore_indices": np.nonzero(mask_i)}),
        "match_ignore_flat_int": lambda: ("match", (init_i.reshape(-1), trg_i.reshape(-1)), {"ignore_indices": idx_i}),
        # NaN in the target; an all-NaN target; shapes that differ with the same size
        "match_nan_target": lambda: ("match", (rain((50, 60), 13), np.where(rain((50, 60), 14) > 3, np.nan,
                                                                            rain((50, 60), 15, dry=0.2))), {}),
        "match_all_nan_target": lambda: ("match", (rain((20, 30), 16), np.full((20, 30), np.nan)), {}),
        "match_shapes_differ": lambda: ("match", (rain((30, 40), 17), rain((40, 30), 18, dry=0.3)), {}),
        "match_all_dry_initial": lambda: ("match", (np.full((20, 20), 0.25), rain((20, 20), 19)), {}),
        "match_all_wet_initial": lambda: ("match", (rain((20, 20), 20, dry=0.0) + 1.0, rain((20, 20), 21)), {}),
        "match_negative_values": lambda: ("match", (rain((30, 30), 22) - 5.0, rain((30, 30), 23, dry=0.2) - 2.0), {}),
        "match_target_inf": lambda: ("match", (rain((30, 30), 24), np.where(rain((30, 30), 25) > 5, np.inf,
                                                                            rain((30, 30), 26))), {}),
        "match_n1": lambda: ("match", (_f([3.0]), _f([7.0])), {}),
        # percentile indices at gamma 0, just below 0.5 and at n - 1
        "match_gamma_zero": lambda: ("match", _gamma_case(101, "zero"), {}),
        "match_gamma_below_half": lambda: ("match", _gamma_case(97, "below_half"), {}),
        "match_percentile_last": lambda: ("match", (_f([5.0] + [0.0] * 9), _f([1, 2, 3, 4, 5, 6, 7, 8, 9, 10])), {}),
        # ties among the wet initial values
        "match_ties_small": lambda: ("match", (tie_init, tie_trg), {}),
        "match_ties_negative_zero": lambda: ("match", (_f([0, 1, 1, 1, 2, 0]), _f([0, -0.0, 0, 3, -0.0, 0])), {}),
        # errors
        "match_error_all_nan": lambda: ("match", (np.full(10, np.nan), np.arange(10.0)), {}),
        "match_error_nonfinite": lambda: ("match", (_f([0, 1, 2, 3, 4] + [np.nan] * 5), np.arange(10.0)), {}),
        "match_error_size": lambda: ("match", (np.arange(10.0), np.arange(12.0)), {}),
        "match_error_empty": lambda: ("match", (np.zeros(0), np.zeros(0)), {}),
        "match_error_ignored_minus_inf": lambda: ("match", (_f([-np.inf, 1, 2, 3]), _f([0, 1, 2, 3])),
                                                  {"ignore_indices": np.array([True, False, False, False])}),
        # resample
        "resample_p0": lambda: ("resample", (rain((40, 40), 31), rain((40, 40), 32), 0.0), {}),
        "resample_p04": lambda: ("resample", (rain((40, 40), 33), rain((40, 40), 34), 0.4), {}),
        "resample_p1": lambda: ("resample", (rain((40, 40), 35), rain((40, 40), 36), 1.0), {}),
        "resample_clip_low": lambda: ("resample", (rain((30, 30), 37), rain((30, 30), 38), -0.5), {}),
        "resample_clip_high": lambda: ("resample", (rain((30, 30), 39), rain((30, 30), 40), 1.5), {}),
        "resample_nan_first": lambda: ("resample", (np.where(rain((30, 30), 41) > 4, np.nan, rain((30, 30), 42)),
                                                    rain((30, 30), 43), 0.6), {}),
        "resample_nan_both_f32": lambda: ("resample", (np.where(rain((30, 30), 44) > 4, np.nan,
                                                                rain((30, 30), 45)).astype(np.float32),
                                                       np.where(rain((30, 30), 46) > 4, np.nan,
                                                                rain((30, 30), 47)).astype(np.float32), 0.3), {}),
        "resample_f32": lambda: ("resample", (rain((30, 30), 48, np.float32), rain((30, 30), 49, np.float32), 0.5), {}),
        "resample_mixed": lambda: ("resample", (rain((30, 30), 50, np.float32), rain((30, 30), 51), 0.5), {}),
        "resample_randomstate": lambda: ("resample", (rain((30, 30), 52), rain((30, 30), 53), 0.7),
                                         {"randgen": "RandomState"}),
        "resample_unit_valid": lambda: ("resample", (_f([1, 3, 5, 7, 9]), _f([2, 4, 6, 8, 10]), 0.6), {}),
        "resample_unit_nan_both": lambda: ("resample", (_f([1, np.nan, np.nan, 7, 9]),
                                                        _f([2.0, 4, np.nan, np.nan, 10]), 1.0), {}),
        "resample_error_shape": lambda: ("resample", (np.zeros(4), np.zeros(5), 0.5), {}),
    }
    return c


CASES = tuple(_cases())


def build_case(name):
    """(fn, args, kwargs) with a live RandomState for a case that names one"""
    fn, args, kw = _cases()[name]()
    if kw.get("randgen") == "RandomState":
        kw = dict(kw, randgen=np.random.RandomState(seed_of(name)))
    return fn, args, kw


def seed_of(name):
    return sum(map(ord, name)) % (2 ** 31)


def sample_index(name, npix):
    """the seeded flat pixel indices stored for a LARGE case"""
    rng = np.random.default_rng(sum(map(ord, name)))
    return np.sort(rng.choice(npix, SAMPLES, replace=False))


def multiset_sha(out):
    """SHA-256 of the output's bit patterns in sorted order: its multiset of values"""
    import hashlib
    a = np.ascontiguousarray(out).reshape(-1)
    it = {4: np.int32, 8: np.int64}[a.dtype.itemsize]
    return hashlib.sha256(np.sort(a.view(it)).tobytes()).hexdigest()


def tie_groups(initial, ignore_indices=None):
    """the groups of wet initial pixels (flat indices) that share a value, for the tie-aware check"""
    x = np.array(initial, dtype=np.float64).reshape(-1)
    mask = np.zeros(np.shape(initial), bool)
    if ignore_indices is not None:
        mask[ignore_indices] = True
    wet = np.flatnonzero(~mask.reshape(-1) & (x > np.nanmin(x)))
    v = x[wet] + 0.0  # -0.0 and +0.0 in one group
    order = np.argsort(v, kind="stable")
    v, wet = v[order], wet[order]
    cuts = np.flatnonzero(np.diff(v) != 0) + 1
    return [g for g in np.split(wet, cuts) if g.size > 1]


def tie_equal(got, want, initial, ignore_indices=None):
    """got equals want bit for bit outside the tie groups, and holds the same values within each; a
    zero may be -0.0 in one and +0.0 in the other (np.nanmin's sign of a zero minimum, and the order
    of -0.0 and +0.0 among equal target values, are NumPy's implementation choices)"""
    g = np.asarray(got, dtype=np.float64).reshape(-1)
    w = np.asarray(want, dtype=np.float64).reshape(-1)
    if g.shape != w.shape:
        return False
    groups = tie_groups(initial, ignore_indices)
    tied = np.zeros(g.size, bool)
    for grp in groups:
        tied[grp] = True
        if not np.array_equal(np.sort(g[grp]), np.sort(w[grp])):
            return False
    gi, wi = g.view(np.int64), w.view(np.int64)
    ok = (gi == wi) | (np.isnan(g) & np.isnan(w)) | ((g == 0) & (w == 0))  # -0.0 against +0.0
    return bool(ok[~tied].all())
