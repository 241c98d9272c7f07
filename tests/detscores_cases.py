"""TEST INFRASTRUCTURE: the deterministic and spatial verification cases shared by the oracle, host-logic
and device tests and the golden generator, and the reference's detcatscores, spatialscores and
ensscores imported through tests/verification_cases.py's stub package."""
import importlib
import warnings

import numpy as np

from verification_cases import rain, reference

MODULES = ("detcatscores", "detcontscores", "spatialscores", "ensscores")


def reference_modules():
    """{name: the reference's module}, or None where the reference is not present"""
    if reference() is None:
        return None
    return {m: importlib.import_module("pysteps.verification." + m) for m in MODULES}


def our_modules():
    from pysteps_b200.verification import detcatscores, detcontscores, ensscores, spatialscores
    return {"detcatscores": detcatscores, "detcontscores": detcontscores, "spatialscores": spatialscores,
            "ensscores": ensscores}


ONLINE = ["ME", "mae", "MSE", "nmse", "rmse", "corr_p", "beta", "beta2", "drmse", "rv"]


def field(rng, shape, dtype=np.float64, nans=0.0, infs=0.0):
    """rain with zeros, NaN and +-inf"""
    X = rain(rng, shape, np.float64, nans=nans)
    u = rng.random(shape)
    X[u < infs / 2] = np.inf
    X[(u >= infs / 2) & (u < infs)] = -np.inf
    return X.astype(dtype)


def numpy_moments(pred, obs, axis, cond, thr):
    """NumPy's own nine np.nanmean results of det_cont_fct_accum over the non-negative axes `axis`, and
    the count of finite residuals"""
    p, o = pred.copy(), obs.copy()
    if cond:
        keep = (o > thr) | (p > thr) if cond == "single" else (o > thr) & (p > thr)
        p[~keep], o[~keep] = np.nan, np.nan
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        res, s = p - o, p + o
        means = [np.nanmean(x, axis=axis) for x in (o, p, res, res ** 2, s ** 2, np.abs(res))]
        mo, mp = means[0], means[1]
        for ax in sorted(axis):
            mo, mp = np.expand_dims(mo, ax), np.expand_dims(mp, ax)
        means += [np.nanmean(x, axis=axis) for x in ((o - mo) * (p - mp), np.abs(o - mo) ** 2, np.abs(p - mp) ** 2)]
    return means, np.sum(np.isfinite(res), axis=axis)


def golden_calls():
    """[(key, module, function, args, kwargs)].  A function ending in "_accum" stands for its *_init(*args[0])
    followed by one accumulation per data tuple in args[1:]; its outcome is the dict."""
    rng = np.random.default_rng(21)
    calls = []
    f32 = np.float32
    # thresholds one float32 ulp either side of a value, as a Python float, an np.float64 and a 0-d array
    v = np.float32(1.3)
    X = np.full((6, 5), v, f32)
    X[::2] = np.nextafter(v, f32(2))
    Y = np.full((6, 5), v, np.float64)
    for i, t in enumerate((float(np.nextafter(v, f32(0))), float(v), float(np.nextafter(v, f32(2))))):
        for kind, thr in (("py", t), ("f64", np.float64(t)), ("arr", np.array(t))):
            calls.append((f"ulp{i}_{kind}/cat", "detcatscores", "det_cat_fct", (X, Y, thr), {}))
            calls.append((f"ulp{i}_{kind}/fss", "spatialscores", "fss", (X, Y, thr, 1), {}))
    # thr - 1 rounding into float32 at 1e8: the non-finite pixels become events
    X = field(rng, (20, 30), f32, nans=0.1, infs=0.1) * f32(1e8)
    calls.append(("big_thr/fss", "spatialscores", "fss", (X, X[::-1].copy(), 1e8, 3), {}))
    calls.append(("big_thr/cat", "detcatscores", "det_cat_fct", (X, X[::-1].copy(), 1e8), {}))
    # axes and shapes for the contingency table
    shapes = [(50,), (7, 9), (4, 6, 5), (3, 1, 4, 5), (1, 8), (2, 3, 1, 6)]
    for shape in shapes:
        A = field(rng, shape, nans=0.05, infs=0.05)
        B = field(rng, shape, f32, nans=0.05, infs=0.05)
        nd = len(shape)
        axes = [None, 0, nd - 1, tuple(range(nd)), -1, (-1, 0), nd, (0, 0)]
        if nd >= 3:
            axes += [(0, 2), (1, nd - 1), (0, 1)]
        for ax in dict.fromkeys(axes):
            calls.append((f"cat{shape}/axis{ax}", "detcatscores", "det_cat_fct", (A, B, 0.5, "", ax), {}))
        calls.append((f"cat{shape}/accum", "detcatscores", "det_cat_fct_accum",
                      ((1.0, 0), (A, B), (B.astype(np.float64), A)), {}))
    # the continuous scores: axes, shapes, conditioning, NaN and +-inf, float32 / float64 mixes
    for shape in [(50,), (7, 9), (4, 6, 5), (3, 1, 4, 5), (1, 8), (2, 3, 1, 6)]:
        for tag, (A, B) in (("inf", (field(rng, shape, nans=0.05, infs=0.05), field(rng, shape, f32, nans=0.05,
                                                                                           infs=0.05))),
                            ("f32", (field(rng, shape, f32, nans=0.05), field(rng, shape, f32, nans=0.05))),
                            ("f64", (field(rng, shape), field(rng, shape, f32)))):
            nd = len(shape)
            axes = [None, 0, nd - 1, tuple(range(nd)), -1, (-1, 0), nd]
            if nd >= 3:
                axes += [(0, 2), (1, nd - 1), (0, 1)]
            if tag != "inf":
                axes.append((0, 0))
            for ax in dict.fromkeys(axes):
                scores = ONLINE if ax in (None, 0) else ["rmse", "corr_p", "beta2"]
                calls.append((f"cont{shape}{tag}/axis{ax}", "detcontscores", "det_cont_fct", (A, B, scores, ax), {}))
            for cond in ("single", "double", "nope"):
                calls.append((f"cont{shape}{tag}/{cond}", "detcontscores", "det_cont_fct",
                              (A, B, ONLINE, 0, cond, 0.5), {}))
            calls.append((f"cont{shape}{tag}/accum", "detcontscores", "det_cont_fct_accum",
                          ((0, None, 0.0), (A, B), (B.astype(np.float64), A)), {}))
    A, B = field(rng, (300, 3), nans=0.05), field(rng, (300, 3), f32, nans=0.05)
    calls.append(("cont/sequential", "detcontscores", "det_cont_fct", (A, B, ONLINE, 0), {}))
    A = field(rng, (6, 7))
    calls.append(("cont/all_nan", "detcontscores", "det_cont_fct", (np.full((6, 7), np.nan), A, ONLINE), {}))
    calls.append(("cont/offline", "detcontscores", "det_cont_fct_compute", (
        {"cov": 1.0, "vobs": 2.0, "vpred": 0.0, "mobs": 1.0, "mpred": 1.0, "me": 0.0, "mse": 1.0, "mss": 0.0,
         "mae": 1.0, "n": 3.0}, ""), {}))
    calls.append(("cont/other_shape", "detcontscores", "det_cont_fct_accum", ((1, None), (A, A), (A[:3], A[:3])), {}))
    calls.append(("cat/all_nan", "detcatscores", "det_cat_fct", (np.full((6, 7), np.nan), A, 0.5), {}))
    calls.append(("cat/other_shape", "detcatscores", "det_cat_fct_accum", ((0.5, None), (A, A), (A[:3], A[:3])), {}))
    calls.append(("cat/shape_mismatch", "detcatscores", "det_cat_fct", (A, A[:3], 0.5), {}))
    calls.append(("cat/scores", "detcatscores", "det_cat_fct", (A, A[::-1].copy(), 0.5, ["csi", "ETS", None, "x"]), {}))
    calls.append(("cat/no_events", "detcatscores", "det_cat_fct", (np.zeros((6, 7)), np.zeros((6, 7)), 0.5), {}))
    # FSS: scales, field shapes, events on neither side
    X = field(rng, (37, 45), nans=0.02, infs=0.02)
    Y = field(rng, (37, 45), f32, nans=0.02)
    for sc in (1, 1.5, 2, 2.5, 3, 16, 60, 200):
        calls.append((f"fss/scale{sc}", "spatialscores", "fss", (X, Y, 1.0, sc), {}))
    for shape in ((1, 40), (40, 1), (1, 1)):
        calls.append((f"fss/{shape}", "spatialscores", "fss", (field(rng, shape), field(rng, shape), 0.5, 5), {}))
    calls.append(("fss/3d", "spatialscores", "fss", (np.zeros((2, 3, 4)), np.zeros((2, 3, 4)), 0.5, 2), {}))
    calls.append(("fss/no_events", "spatialscores", "fss", (np.zeros((9, 8)), np.zeros((9, 8)), 0.5, 3), {}))
    calls.append(("fss/accum_twice", "spatialscores", "fss_accum", ((1.0, 4), (X, Y), (Y, X)), {}))
    empty = {"thr": 1.0, "scale": 2, "sum_fct_sq": 0.0, "sum_fct_obs": 0.0, "sum_obs_sq": 0.0}
    calls.append(("fss/never_accumulated", "spatialscores", "fss_compute", (empty,), {}))
    calls.append(("intensity_scale", "spatialscores", "intensity_scale", (X, Y, "FSS", [2.0, 0.5, 1.0], [8, 1, 3]), {}))
    calls.append(("intensity_scale/no_scales", "spatialscores", "intensity_scale", (X, Y, "fss", 1.0), {}))
    calls.append(("intensity_scale/unknown", "spatialscores", "intensity_scale", (X, Y, "nope", 1.0, 2), {}))
    # ensemble skill and spread
    E = field(rng, (5, 30, 26), nans=0.02)
    o = field(rng, (30, 26), f32)
    for metric, kw in (("fss", dict(thr=1.0, scale=5)), ("fss", dict(thr=0.5, scale=1)), ("CSI", dict(thr=1.0)),
                       ("csi", dict(thr=1.0)), ("POD", dict(thr=0.5)), ("nope", dict(thr=1.0)),
                       ("fss", dict(thr=1.0)), ("RMSE", {}), ("rmse", {}), ("beta", {}), ("corr_p", {"axis": 1}),
                       ("ME", {"conditioning": "double", "thr": 0.5})):
        tag = f"{metric}{sorted(kw)}{kw.get('scale')}"
        calls.append((f"skill/{tag}", "ensscores", "ensemble_skill", (E, o, metric), kw))
        calls.append((f"spread/{tag}", "ensscores", "ensemble_spread", (E, metric), kw))
    calls.append(("spread/k1", "ensscores", "ensemble_spread", (E[:1], "fss"), dict(thr=1.0, scale=2)))
    calls.append(("skill/2d", "ensscores", "ensemble_skill", (o, o, "fss"), dict(thr=1.0, scale=2)))
    calls.append(("skill/mismatch", "ensscores", "ensemble_skill", (E, o[:5], "fss"), dict(thr=1.0, scale=2)))
    return calls


def run_call(mod, fn, args, kwargs):
    """(outcome, ["Category: message", ...]) of one call of the module mod"""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            if fn.endswith("_accum"):
                d = getattr(mod, fn.replace("_accum", "_init"))(*args[0])
                for data in args[1:]:
                    getattr(mod, fn)(d, *data)
                out = d
            else:
                out = getattr(mod, fn)(*args, **kwargs)
        except Exception as e:  # noqa: BLE001 -- the exception is the outcome
            out = e
    return out, [f"{x.category.__name__}: {x.message}" for x in w]
