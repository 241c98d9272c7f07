"""CPU test of the HOST logic of pysteps_b200.blending (metadata, shape flow, member maps, errors, dtypes)
and of pysteps_b200.nowcasts.extrapolation, with the entry points emulated (tests/cpu_abi_blending.py),
against the live reference on randomised valid and invalid calls: exceptions and their messages,
shapes, dtypes and values."""
import contextlib
import io

import numpy as np
import pytest

import cpu_abi_blending
from conftest import bits_equal


def _reference(name="pysteps.blending.linear_blending"):
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    return _refimport.ref_module(name)


def _outcome(fn, *a, **k):
    try:
        with np.errstate(all="ignore"):
            return fn(*a, **k)
    except Exception as e:  # noqa: BLE001 -- the exception is the result
        return e


def _same(got, want):
    if isinstance(want, ValueError) and str(want).startswith("Unknown method "):
        # pysteps_b200.extrapolation.get_method lists its "semilagrangian_b200" among the available names
        return isinstance(got, ValueError) and str(got).split("\n")[0] == str(want).split("\n")[0], (got, want)
    if isinstance(want, Exception):
        return isinstance(got, type(want)) and str(got) == str(want), (repr(got), repr(want))
    if isinstance(got, Exception):
        return False, (repr(got), repr(want))
    return bits_equal(np.asarray(got), want), (np.shape(got), np.asarray(got).dtype, want.shape, want.dtype)


_METAS = [
    {"unit": "mm/h", "transform": None},
    {"unit": "mm/h", "transform": "dB", "threshold": -10.0, "zerovalue": -15.0},
    {"unit": "mm/h", "transform": "dB"},
    {"unit": "mm/h", "transform": "sqrt", "threshold": 0.3, "zerovalue": 0.0},
    {"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": 0.0, "threshold": -2.0},
    {"unit": "mm/h", "transform": "log", "threshold": -2.0},
    {"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": 0.5, "threshold": -1.0},
    {"unit": "mm", "transform": None, "accutime": 5, "threshold": 0.1, "zerovalue": 0.0},
    {"unit": "mm", "transform": "sqrt", "accutime": 10.0, "threshold": 0.1, "zerovalue": 0.0},
    {"unit": "dBZ", "transform": None, "threshold": 0.1, "zerovalue": 0.0},
    {"unit": "dBZ", "transform": None, "threshold": 0.1, "zerovalue": 0.0, "zr_a": 316.0, "zr_b": 1.5},
    {"unit": "mm", "transform": None, "threshold": 0.1, "zerovalue": 0.0},       # KeyError accutime
    {"unit": "mm/h"},                                                            # KeyError transform
    {"transform": None},                                                         # KeyError unit
    {"unit": "inch", "transform": None},                                         # ValueError unit
    {"unit": "mm/h", "transform": "cubic"},                                      # ValueError transform
]


def _random_call(rng):
    dt = [np.float32, np.float64][int(rng.integers(2))]
    m, n = int(rng.integers(3, 9)), int(rng.integers(3, 9))
    if rng.random() < 0.05:
        m = 1
    meta_now = dict(_METAS[int(rng.integers(len(_METAS)))]) if rng.random() < 0.5 else dict(_METAS[0])
    meta_nwp = dict(_METAS[int(rng.integers(len(_METAS)))]) if rng.random() < 0.3 else dict(_METAS[0])
    if meta_now.get("transform") in ("dB",):
        P = rng.uniform(-20, 15, (m, n))
    elif meta_now.get("transform") in ("BoxCox", "log"):
        P = rng.uniform(-3, 2, (m, n))
    elif meta_now.get("unit") == "dBZ":
        P = rng.uniform(0, 50, (m, n))
    else:
        P = np.where(rng.random((m, n)) < 0.4, 0.0, rng.gamma(0.8, 2.0, (m, n)))
    P[rng.random((m, n)) < 0.1] = np.nan
    if rng.random() < 0.1:
        P[rng.random((m, n)) < 0.1] = np.inf  # can make a diff of NaN: scipy's all-NaN rank
    if rng.random() < 0.2:
        P = np.repeat(P[None], 3, axis=0)  # 3-D precip: the last frame is used
    P = P.astype(dt)
    timestep = [5, 10, 3, 7][int(rng.integers(4))]
    timesteps = int(rng.integers(1, 9))
    start = int(rng.integers(0, 40))
    end = start + int(rng.integers(1, 60))
    k = [0, 1, 1, 3, 10, -1][int(rng.integers(6))]
    T_nwp = timesteps if rng.random() < 0.8 else int(rng.integers(1, 10))
    if k == 0:
        R = None
    else:
        shape = (T_nwp, m, n) if k == -1 else (k, T_nwp, m, n)
        if rng.random() < 0.05:
            shape = shape[:-1] + (n + 1,)  # grid mismatch: the AssertionError
        R = np.where(rng.random(shape) < 0.4, 0.0, rng.gamma(0.8, 2.0, shape))
        u = rng.random(shape)
        R[u < 0.05] = np.nan
        R[(u > 0.05) & (u < 0.07)] = np.inf
        R[(u > 0.07) & (u < 0.08)] = -np.inf
        if rng.random() < 0.05:
            R[:] = 0.0
        R = R.astype([np.float32, np.float64][int(rng.integers(2))] if rng.random() < 0.3 else dt)
    method = ["eulerian", "eulerian", "extrapolation", "lagrangian", "no_such_nowcast"][int(rng.integers(5))]
    V = rng.uniform(-1.5, 1.5, (2, m, n)) if method != "eulerian" else np.zeros((2, m, n))
    kw = dict(start_blending=start, end_blending=end, fill_nwp=bool(rng.random() < 0.7),
              saliency=bool(rng.random() < 0.5))
    return (P, meta_now, V, timesteps, timestep, method, R, meta_nwp), kw


def test_random_calls_match_the_reference():
    lb = _reference()
    import pysteps_b200.blending.linear_blending as ours
    rng = np.random.default_rng(20261017)
    compared = errors = nie = 0
    for it in range(160):
        args, kw = _random_call(rng)
        want = _outcome(lb.forecast, *[a.copy() if isinstance(a, np.ndarray) else a for a in args], **kw)
        with cpu_abi_blending.emulated():
            got = _outcome(ours.forecast, *args, **kw)
        if isinstance(got, NotImplementedError):
            nie += 1
            continue
        ok, info = _same(got, want)
        assert ok, (it, info)
        compared += 1
        errors += isinstance(want, Exception)
    assert compared >= 100 and errors >= 20, (compared, errors, nie)


def test_fixup_path_runs_and_decides_as_numpy():
    lb = _reference()
    import pysteps_b200.blending.linear_blending as ours
    P = np.full((4, 5), -10.0)  # 10 ** (-10 / 10) is the threshold itself
    P[0, 0] = np.nextafter(-10.0, 0)
    R = np.ones((3, 4, 5))
    meta = {"unit": "mm/h", "transform": "dB", "threshold": -10.0}
    args = (P, meta, np.zeros((2, 4, 5)), 3, 10, "eulerian", R, {"unit": "mm/h", "transform": None})
    want = lb.forecast(*args, start_blending=0, end_blending=20)
    cpu_abi_blending.fixups.clear()
    with cpu_abi_blending.emulated():
        got = ours.forecast(*args, start_blending=0, end_blending=20)
    assert cpu_abi_blending.fixups[0] == 2 * 20  # every pixel of both nowcast leads
    assert bits_equal(got, want)


def test_nowcast_method_lookup():
    lb = _reference()
    import pysteps_b200.blending.linear_blending as ours
    P = np.ones((4, 5))
    args = (P, {"unit": "mm/h", "transform": None}, np.zeros((2, 4, 5)), 2, 10, 7, None, None)
    want = _outcome(lb.forecast, *args)
    with cpu_abi_blending.emulated():
        got = _outcome(ours.forecast, *args)
    assert _same(got, want)[0], (got, want)


# ---------------------------------------------------------------- the extrapolation nowcast
def _random_nowcast_call(rng):
    m, n = int(rng.integers(3, 9)), int(rng.integers(3, 9))
    P = rng.gamma(0.8, 2.0, (m, n)).astype([np.float32, np.float64][int(rng.integers(2))])
    if rng.random() < 0.3:
        P[rng.random((m, n)) < 0.2] = np.nan
    V = rng.uniform(-2, 2, (2, m, n))
    r = rng.random()
    if r < 0.08:
        P = P[0]                       # 1-D precip
    elif r < 0.16:
        V = V[0]                       # 2-D velocity
    elif r < 0.24:
        V = rng.uniform(-2, 2, (2, m + 1, n))  # shape mismatch
    timesteps = [int(rng.integers(1, 5)), [1, 2, 3.5], [2, 1], [0.5]][int(rng.integers(4))]
    kw = {}
    if rng.random() < 0.3:
        kw["extrap_method"] = ["eulerian", "semilagrangian", "nope"][int(rng.integers(3))]
    if rng.random() < 0.3:
        kw["extrap_kwargs"] = {"outval": 0.0}
    return (P, V, timesteps), kw


def test_extrapolation_nowcast_matches_the_reference():
    ref = _reference("pysteps.nowcasts.extrapolation")
    from pysteps_b200.nowcasts import extrapolation as ours
    rng = np.random.default_rng(5)
    compared = errors = 0
    for it in range(120):
        args, kw = _random_nowcast_call(rng)
        want = _outcome(ref.forecast, *args, **kw)
        with cpu_abi_blending.emulated():
            got = _outcome(ours.forecast, *args, **kw)
        ok, info = _same(got, want)
        assert ok, (it, kw, info)
        compared += 1
        errors += isinstance(want, Exception)
    assert compared >= 100 and errors >= 20, (compared, errors)


def test_extrapolation_nowcast_measure_time():
    ref = _reference("pysteps.nowcasts.extrapolation")
    from pysteps_b200.nowcasts import extrapolation as ours
    rng = np.random.default_rng(1)
    P, V = rng.gamma(0.8, 2.0, (6, 7)), rng.uniform(-1, 1, (2, 6, 7))
    outs = []
    for fn, ctx in ((ref.forecast, contextlib.nullcontext()), (ours.forecast, cpu_abi_blending.emulated())):
        buf = io.StringIO()
        with ctx, contextlib.redirect_stdout(buf):
            F, t = fn(P, V, 3, measure_time=True)
        outs.append((F, buf.getvalue().split("...")[0], isinstance(t, float)))
    assert bits_equal(outs[0][0], outs[1][0]) and outs[0][1:] == outs[1][1:]
