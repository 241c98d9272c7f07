"""TEST INFRASTRUCTURE: the verification cases shared by the oracle, host-logic and device tests, and
the reference's verification modules imported without ``pysteps/verification/__init__.py`` (it
imports the plots and so matplotlib): a stub namespace package over the reference's directory."""
import importlib
import os
import sys
import types

import numpy as np


def reference():
    """(probscores, ensscores) of the reference, or None where it is not present"""
    import _refimport
    if not _refimport.available():
        return None
    pk = _refimport.import_reference()
    if "pysteps.verification" not in sys.modules:
        vm = types.ModuleType("pysteps.verification")
        vm.__path__ = [os.path.join(r, "verification") for r in pk.__path__]
        sys.modules["pysteps.verification"] = vm
        pk.verification = vm
    return (importlib.import_module("pysteps.verification.probscores"),
            importlib.import_module("pysteps.verification.ensscores"))


def rain(rng, shape, dtype=np.float64, zeros=0.5, nans=0.0):
    """gamma rain with exact zeros and some NaN"""
    X = np.where(rng.random(shape) < zeros, 0.0, rng.gamma(0.6, 2.0, shape))
    if nans:
        X[rng.random(shape) < nans] = np.nan
    return X.astype(dtype)


def ensemble_cases():
    """name -> (X_f, X_o, X_min) for CRPS and the rank histogram"""
    rng = np.random.default_rng(11)
    out = {}
    for k in (1, 2, 7, 8, 9, 127, 128, 129, 300):
        out[f"k{k}"] = (rain(rng, (k, 6, 7), nans=0.01), rain(rng, (6, 7)), 0.1)
    for n in (0, 7, 8, 128, 129, 255, 256, 257, 1000, 4099):
        X = rng.normal(size=(5, n)).astype(np.float64)
        out[f"pixels{n}"] = (X, rng.normal(size=n), None)
    X = rng.normal(size=(4, 30))
    out["all_nan"] = (np.full((4, 30), np.nan), X[0], None)
    out["zeros_min"] = (rain(rng, (6, 40, 30), zeros=0.8), rain(rng, (40, 30), zeros=0.8), 0.1)
    out["zeros_nomin"] = (rain(rng, (6, 40, 30), zeros=0.8), rain(rng, (40, 30), zeros=0.8), None)
    X = np.round(rng.normal(size=(9, 50, 20)) * 2) / 2
    out["obs_on_members"] = (X, X[3].copy(), None)
    X = rain(rng, (8, 33, 31), np.float32, zeros=0.6)
    out["f32_f64_half"] = (X, rain(rng, (33, 31), np.float64, zeros=0.6), 0.5)
    out["f32_f64_tenth"] = (X, rain(rng, (33, 31), np.float64, zeros=0.6), 1.1)
    out["f64_f32"] = (rain(rng, (8, 33, 31), zeros=0.3), rain(rng, (33, 31), np.float32, zeros=0.3), np.float32(0.1))
    out["f32_f32"] = (X, rain(rng, (33, 31), np.float32, zeros=0.6), 0.1)
    X = np.zeros((6, 10, 10))
    X[:, ::2] = -0.0
    out["signed_zeros"] = (X, np.where(rng.random((10, 10)) < 0.5, -0.0, 0.0), None)
    # +0 and -0 members on both sides of nonzero observations: the sort may put either zero first
    v = np.array([-0.0, 0.0, -0.0, 0.0, -1.0, 1.0, 0.5])
    out["signed_zeros_mixed"] = (v[rng.integers(0, 7, (7, 30, 20))],
                                 np.array([0.25, -0.5, 0.0, -0.0, 1.0, -2.0])[rng.integers(0, 6, (30, 20))], None)
    X = v[rng.integers(0, 7, (7, 30, 20))].astype(np.float32)
    out["signed_zeros_mixed_f32"] = (X, np.array([0.25, -0.5, 0.0, 3.0], np.float32)[rng.integers(0, 4, (30, 20))],
                                     0.0)
    return out


def flip_zeros(X):
    """X with the sign of every zero flipped"""
    return np.where(X == 0, np.where(np.signbit(X), X.dtype.type(0.0), X.dtype.type(-0.0)), X).astype(X.dtype)


def prob_cases():
    """name -> (P_f, X_o, X_min, n) for reldiag (n bins) and the ROC curve (n thresholds)"""
    rng = np.random.default_rng(12)
    out = {}
    for n in (1, 2, 10, 101):
        P = (rng.integers(0, 25, (40, 50)) / 24.0)
        out[f"n{n}"] = (P, rain(rng, (40, 50), nans=0.02), 0.5, n)
        out[f"n{n}_f32"] = (P.astype(np.float32), rain(rng, (40, 50), np.float32), 0.1, n)
    edges = np.linspace(-1e-6, 1 + 1e-6, 11)
    P = np.concatenate([edges, np.linspace(0, 1, 10), np.linspace(0, 1, 101), [np.nan, np.inf]])
    out["on_edges"] = (P, rng.gamma(1.0, 1.0, P.shape), 1.0, 10)
    out["on_edges_101"] = (P, rng.gamma(1.0, 1.0, P.shape), 1.0, 101)
    out["empty"] = (np.zeros(0), np.zeros(0), 1.0, 10)
    out["large"] = (rng.random((3, 300, 301)), rain(rng, (3, 300, 301)), 0.5, 10)
    return out


def golden_calls():
    """[(key, module "probscores" | "ensscores", function, args, seed or None)]: the calls the goldens
    record.  A function ending in "_accum" stands for its *_init(*init_args) followed by the
    accumulation of the data; its outcome is the dict."""
    from oracle import verification as ora
    calls = []
    for name, (X_f, X_o, X_min) in sorted(ensemble_cases().items()):
        k = X_f.shape[0]
        calls.append((f"{name}/CRPS", "probscores", "CRPS", (X_f, X_o), None))
        calls.append((f"{name}/CRPS_accum", "probscores", "CRPS_accum", ((), X_f, X_o), None))
        for tag, xm in (("nomin", None), ("min", X_min)):
            seed = 1000 + len(calls)
            calls.append((f"{name}/rankhist_{tag}", "ensscores", "rankhist", (X_f, X_o, xm, False), seed))
            calls.append((f"{name}/rankhist_{tag}_norm", "ensscores", "rankhist", (X_f, X_o, xm), seed))
            calls.append((f"{name}/rankhist_{tag}_accum", "ensscores", "rankhist_accum", ((k, xm), X_f, X_o), seed))
    for name, (P, O, X_min, nb) in sorted(prob_cases().items()):
        count = ora.reldiag(P, O, X_min, np.linspace(-1e-6, 1 + 1e-6, nb + 1))[0]
        top = int(count.max()) if count.size else 0
        for mc in sorted({0, 10, top, top + 1}):
            calls.append((f"{name}/reldiag_{mc}", "probscores", "reldiag", (P, O, X_min, nb, mc), None))
            calls.append((f"{name}/reldiag_{mc}_accum", "probscores", "reldiag_accum", ((X_min, nb, mc), P, O), None))
        for area in (False, True):
            calls.append((f"{name}/ROC_{area}", "probscores", "ROC_curve", (P, O, X_min, nb, area), None))
        calls.append((f"{name}/ROC_accum", "probscores", "ROC_curve_accum", ((X_min, nb), P, O), None))
    return calls


def run_call(mod, fn, args, seed):
    """(outcome, ["Category: message", ...], next np.random.random()) of one golden call of the module
    mod (a probscores or an ensscores)"""
    import warnings
    if seed is not None:
        np.random.seed(seed)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            if fn.endswith("_accum"):
                init = getattr(mod, fn.replace("_accum", "_init"))
                d = init(*args[0])
                getattr(mod, fn)(d, *args[1:])
                out = d
            else:
                out = getattr(mod, fn)(*args)
        except Exception as e:  # noqa: BLE001 -- the exception is the outcome
            out = e
    return out, [f"{x.category.__name__}: {x.message}" for x in w], np.random.random()


def encode(out):
    """(signature string, uint8 bytes) of an outcome: its Python/NumPy types and shapes (or the
    exception and its message), and its values bit for bit"""
    arrays = []

    def enc(x):
        if isinstance(x, Exception):
            return f"{type(x).__name__}({x})"
        if isinstance(x, dict):
            return "{" + ",".join(f"{k}:{enc(x[k])}" for k in x) + "}"
        if isinstance(x, (tuple, list)):
            return type(x).__name__ + "[" + ",".join(enc(v) for v in x) + "]"
        if x is None:
            return "None"
        a = np.asarray(x)
        arrays.append(np.ascontiguousarray(a).tobytes())
        return f"{type(x).__name__}:{a.dtype}{list(a.shape)}"
    sig = enc(out)
    return sig, np.frombuffer(b"".join(arrays), dtype=np.uint8)


def same_outcome(a, b):
    """equal signatures and bit-identical values"""
    (sa, xa), (sb, xb) = encode(a), encode(b)
    return sa == sb and xa.tobytes() == xb.tobytes()


class Goldens:
    """tests/golden/verification_golden.npz by call key"""

    def __init__(self, path):
        g = np.load(path)
        self.sig, self.vals, self.off = g["sig"], g["vals"], g["off"]
        self.warnings, self.next = g["warnings"], g["next"]
        self.index = {str(k): i for i, k in enumerate(g["keys"])}

    def outcome(self, key):
        """(signature, bytes, warnings, next draw or None) stored for a call"""
        i = self.index[key]
        w = str(self.warnings[i])
        return (str(self.sig[i]), self.vals[self.off[i]:self.off[i + 1]].tobytes(), w.split("\n") if w else [],
                None if np.isnan(self.next[i]) else float(self.next[i]))


def matches_golden(g, key, out, warned, nxt):
    sig, vals, w, n = g.outcome(key)
    s, v = encode(out)
    problems = []
    if s != sig:
        problems.append(f"types {s} != {sig}")
    elif v.tobytes() != vals:
        problems.append("values differ")
    if warned != w:
        problems.append(f"warnings {warned} != {w}")
    if n is not None and nxt != n:
        problems.append("the random state after the call differs")
    return problems
