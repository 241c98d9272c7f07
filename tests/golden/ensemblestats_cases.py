"""Inputs of the ensemble-statistics goldens (tests/golden/ensemblestats_golden.npz), shared by the
generator, the CPU tests and the GPU tests.  build_case(name) -> (function name, args, kwargs) of
``mean(X, ...)``, ``excprob(X, X_thr, ...)`` or ``banddepth(X, ...)``; banddepth cases also have a
seed (seed_of) for np.random.seed before the call.

Cases of up to 2^16 values per output store the reference's whole output; LARGE cases store SAMPLES
seeded pixels of every output plane and each plane's NaN count."""
import numpy as np

SAMPLES = 2048
LARGE = ("mean_f32_24x512", "excprob_f64_24x512_4thr", "excprob_f32_24x512_ignore_nan")
F32_TENTH = float(np.float32(0.1))
ABOVE = float(np.nextafter(np.float32(0.1), np.float32(1)))  # the next float32 after 0.1f, as a float
WEAK_ABOVE = F32_TENTH + 1e-12  # rounds to 0.1f in float32, but lies above it in float64


def rain(k, shape, seed, dtype=np.float64, zeros=0.5):
    """k members of rain-like values, `zeros` of them exactly 0 (ties for banddepth)"""
    rng = np.random.default_rng(seed)
    X = rng.gamma(0.8, 2.0, (k,) + tuple(shape))
    X[rng.random(X.shape) < zeros] = 0.0
    return X.astype(dtype)


def tenths(k, shape, seed, dtype=np.float32):
    """values that are exactly float32(0.1), its neighbours or 0, for threshold-rounding cases"""
    rng = np.random.default_rng(seed)
    v = np.array([0.0, np.nextafter(np.float32(0.1), np.float32(0)), np.float32(0.1), np.float32(ABOVE)],
                 dtype=np.float32)
    return v[rng.integers(0, 4, (k,) + tuple(shape))].astype(dtype)


def nonfinite(X, seed, frac=0.05, all_nan_pixels=3):
    """NaN, +inf and -inf members at seeded places, and a few pixels where every member is NaN"""
    rng = np.random.default_rng(seed)
    X = X.copy()
    u = rng.random(X.shape)
    X[u < frac / 3] = np.nan
    X[(u >= frac / 3) & (u < 2 * frac / 3)] = np.inf
    X[(u >= 2 * frac / 3) & (u < frac)] = -np.inf
    flat = X.reshape(X.shape[0], -1)
    flat[:, rng.choice(flat.shape[1], all_nan_pixels, replace=False)] = np.nan
    return X


def nan_only(X, seed, frac=0.1):
    rng = np.random.default_rng(seed)
    X = X.copy()
    X[rng.random(X.shape) < frac] = np.nan
    return X


def _neg_zero(X):
    X = X.copy()
    X[X == 0] = -0.0
    return X


def _cases():
    c = {
        # mean
        "mean_f64_24": lambda: ("mean", (rain(24, (40, 56), 1),), {}),
        "mean_f32_24": lambda: ("mean", (rain(24, (40, 56), 2, np.float32),), {}),
        "mean_f64_nan_inf": lambda: ("mean", (nonfinite(rain(24, (32, 40), 3), 3),), {}),
        "mean_f32_ignore_nan": lambda: ("mean", (nonfinite(rain(24, (32, 40), 4, np.float32), 4),),
                                        {"ignore_nan": True}),
        "mean_f64_ignore_nan_nan_only": lambda: ("mean", (nan_only(rain(12, (30, 20), 5), 5, 0.3),),
                                                 {"ignore_nan": True}),
        "mean_f64_xthr": lambda: ("mean", (rain(24, (32, 48), 6),), {"X_thr": 0.1}),
        "mean_f32_xthr_weak": lambda: ("mean", (tenths(24, (32, 40), 7),), {"X_thr": WEAK_ABOVE}),
        "mean_f32_xthr_strong": lambda: ("mean", (tenths(24, (32, 40), 7),), {"X_thr": np.float64(WEAK_ABOVE)}),
        "mean_f32_xthr_nan": lambda: ("mean", (nonfinite(rain(16, (24, 24), 8, np.float32), 8),), {"X_thr": 0.5}),
        "mean_2d": lambda: ("mean", (rain(1, (40, 30), 9)[0],), {}),
        "mean_2d_negative_zero": lambda: ("mean", (_neg_zero(rain(1, (16, 16), 10)[0]),), {}),
        "mean_k0": lambda: ("mean", (np.zeros((0, 6, 7)),), {}),
        "mean_k0_ignore_nan": lambda: ("mean", (np.zeros((0, 6, 7), np.float32),), {"ignore_nan": True}),
        "mean_k1": lambda: ("mean", (rain(1, (20, 24), 11),), {}),
        "mean_k2": lambda: ("mean", (rain(2, (20, 24), 12, np.float32),), {}),
        "mean_k130": lambda: ("mean", (rain(130, (16, 20), 13, np.float32),), {}),
        "mean_f32_overflow": lambda: ("mean", (np.full((3, 4, 5), 2e38, np.float32),), {}),
        "mean_1xn": lambda: ("mean", (rain(24, (1, 97), 14),), {}),
        "mean_mx1": lambda: ("mean", (rain(24, (97, 1), 15, np.float32),), {"ignore_nan": True}),
        "mean_f32_24x512": lambda: ("mean", (rain(24, (512, 512), 16, np.float32),), {}),
        # excprob
        "excprob_f64_scalar": lambda: ("excprob", (rain(24, (40, 56), 21), 1.0), {}),
        "excprob_f32_list_weak": lambda: ("excprob", (tenths(24, (32, 40), 22), [WEAK_ABOVE, F32_TENTH, 0.0]), {}),
        "excprob_f32_ndarray_strong": lambda: ("excprob", (tenths(24, (32, 40), 22),
                                                           np.array([WEAK_ABOVE, F32_TENTH, 0.0])), {}),
        "excprob_f32_np_float64": lambda: ("excprob", (tenths(24, (32, 40), 23), np.float64(WEAK_ABOVE)), {}),
        "excprob_f32_above": lambda: ("excprob", (tenths(24, (32, 40), 24), ABOVE), {}),
        "excprob_f64_nonfinite": lambda: ("excprob", (nonfinite(rain(24, (32, 40), 25), 25), [0.5, 2.0]), {}),
        "excprob_f64_nonfinite_ignore_nan": lambda: ("excprob", (nonfinite(rain(24, (32, 40), 25), 25), [0.5, 2.0]),
                                                     {"ignore_nan": True}),
        "excprob_4d": lambda: ("excprob", (rain(12, (3, 16, 20), 26), [0.1, 1.0, 5.0]), {}),
        "excprob_k0": lambda: ("excprob", (np.zeros((0, 5, 6)), [0.5, 1.0]), {}),
        "excprob_k0_ignore_nan": lambda: ("excprob", (np.zeros((0, 5, 6)), 0.5), {"ignore_nan": True}),
        "excprob_k1": lambda: ("excprob", (rain(1, (20, 24), 27), 0.5), {}),
        "excprob_k2": lambda: ("excprob", (rain(2, (20, 24), 28, np.float32), 0.5), {}),
        "excprob_k130": lambda: ("excprob", (rain(130, (16, 20), 29), [0.1, 1.0]), {}),
        "excprob_nine_thresholds": lambda: ("excprob", (rain(24, (24, 32), 30), list(np.linspace(0, 4, 9))), {}),
        "excprob_1xn": lambda: ("excprob", (rain(24, (1, 97), 31), 0.5), {}),
        "excprob_mx1": lambda: ("excprob", (rain(24, (97, 1), 32, np.float32), [0.5, np.inf]), {}),
        "excprob_f64_24x512_4thr": lambda: ("excprob", (rain(24, (512, 512), 33), [0.1, 0.5, 1.0, 5.0]), {}),
        "excprob_f32_24x512_ignore_nan": lambda: ("excprob", (nonfinite(rain(24, (512, 512), 34, np.float32), 34),
                                                              [0.1, 0.5, 1.0, 5.0]), {"ignore_nan": True}),
        # banddepth
        "banddepth_f64": lambda: ("banddepth", (rain(24, (32, 40), 41),), {}),
        "banddepth_f32_ties": lambda: ("banddepth", (rain(24, (48, 40), 42, np.float32, zeros=0.8),), {}),
        "banddepth_thr": lambda: ("banddepth", (rain(24, (32, 40), 43),), {"thr": 1.0}),
        "banddepth_norm": lambda: ("banddepth", (rain(24, (32, 40), 44),), {"norm": True}),
        "banddepth_nan": lambda: ("banddepth", (nonfinite(rain(12, (32, 40), 45), 45),), {}),
        "banddepth_all_nan": lambda: ("banddepth", (np.full((4, 5, 6), np.nan),), {}),
        "banddepth_p0": lambda: ("banddepth", (rain(8, (16, 16), 46),), {"thr": 1e9}),
        "banddepth_k1": lambda: ("banddepth", (rain(1, (16, 16), 47),), {}),
        "banddepth_k2": lambda: ("banddepth", (rain(2, (16, 16), 48),), {}),
        "banddepth_k130": lambda: ("banddepth", (rain(130, (12, 16), 49, np.float32),), {}),
        "banddepth_3d_pixels": lambda: ("banddepth", (rain(10, (3, 8, 9), 50),), {"thr": np.float64(0.5)}),
        "banddepth_2d_members": lambda: ("banddepth", (rain(16, (300,), 51),), {}),
        "banddepth_f32_24x256": lambda: ("banddepth", (rain(24, (256, 256), 52, np.float32),), {}),
    }
    return c


CASES = tuple(_cases())


def build_case(name):
    return _cases()[name]()


def seed_of(name):
    """the np.random.seed of a banddepth case"""
    return sum(map(ord, name)) % (2 ** 31)


def sample_index(name, npix):
    """the seeded flat pixel indices stored for a LARGE case"""
    rng = np.random.default_rng(sum(map(ord, name)))
    return np.sort(rng.choice(npix, SAMPLES, replace=False))
