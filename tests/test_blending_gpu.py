"""GPU: linear and salient blending (csrc/blending.cu) against oracle/blending.py, bit for bit where
the conversion is exact; the dense rank against np.unique; NumPy against CUDA-tensor input; repeated
calls; the threshold fix-up of the dB conversion."""
import numpy as np
import pytest
import torch

from conftest import bits_equal
from oracle import blending as ora
from test_oracle_blending import CASES, make_case

pytestmark = pytest.mark.gpu


def _ours():
    from pysteps_b200.blending import linear_blending
    return linear_blending


def _run(P, R, sal, fill, meta=None, T=6):
    return _ours().forecast(P, meta or {"unit": "mm/h", "transform": None}, np.zeros((2,) + P.shape[-2:]), T, 10,
                            "eulerian", R, {"unit": "mm/h", "transform": None}, start_blending=10, end_blending=40,
                            fill_nwp=fill, saliency=sal)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_device_equals_oracle(case):
    c = CASES[case]
    P, R = make_case(c["seed"], n_nwp=c["n_nwp"], dt=c["dt"], special=c["special"])
    got = _run(P, R, c["saliency"], c["fill"])
    with np.errstate(all="ignore"):
        want = ora.blend(np.repeat(P[None], 4, axis=0), R, 6, 10, 10, 40, c["fill"], c["saliency"])
    assert bits_equal(got, want)


@pytest.mark.parametrize("n_now,n_nwp", [(10, 3), (3, 10), (3, 1), (1, 1)])
@pytest.mark.parametrize("sal", [False, True])
def test_member_maps_and_mixed_dtypes(n_now, n_nwp, sal):
    rng = np.random.default_rng(n_now * 11 + n_nwp)
    P, R = make_case(5, n_nwp=n_nwp, dt=np.float64, nwp_dt=np.float32)
    now = rng.gamma(0.8, 2.0, (n_now, 4) + P.shape).astype(np.float32) if n_now > 1 else None
    import pysteps_b200.nowcasts.interface as ni
    ni._nowcast_methods["_test_ensemble"] = lambda p, v, t, **k: now[:, :t] if now is not None else \
        np.repeat(np.float32(p)[None], t, axis=0)
    try:
        got = _ours().forecast(P, {"unit": "mm/h", "transform": None}, np.zeros((2,) + P.shape), 6, 10,
                               "_test_ensemble", R, {"unit": "mm/h", "transform": None}, start_blending=10,
                               end_blending=40, saliency=sal)
    finally:
        del ni._nowcast_methods["_test_ensemble"]
    src = now if now is not None else np.repeat(np.float32(P)[None], 4, axis=0)
    with np.errstate(all="ignore"):
        want = ora.blend(src, R, 6, 10, 10, 40, True, sal)
    assert bits_equal(got, want)


def test_sqrt_and_mm_are_exact():
    P, R = make_case(3, n_nwp=3)
    P = np.abs(P)
    meta = {"unit": "mm", "transform": "sqrt", "accutime": 5, "threshold": 0.1, "zerovalue": 0.0}
    got = _run(P, R, True, True, meta=meta)
    want = ora.blend(np.repeat(ora.to_rainrate(P, meta)[None], 4, axis=0), R, 6, 10, 10, 40, True, True)
    assert bits_equal(got, want)


def _convert(x, meta):
    """the device conversion and the number of pixels it left to the host's fix-up"""
    from unittest import mock
    from pysteps_b200 import _lib
    from pysteps_b200.blending.linear_blending import to_rainrate
    fixed = []
    real = _lib.call

    def spy(name, *args):
        if name == "b200_blend_scatter":
            fixed.append(args[4])
        return real(name, *args)

    with mock.patch.object(_lib, "call", spy):
        got, _ = to_rainrate(torch.from_numpy(x).cuda(), meta)
    return got.cpu().numpy(), sum(fixed)


def _bound_ulps(kind_z):
    return 16.0 * (2.0 + kind_z)


_CONVERSIONS = [
    # (metadata, input range, threshold in the transformed unit or None, per-pixel exponent for the bound)
    ({"unit": "mm/h", "transform": "dB", "threshold": -10.0}, (-20, 20), -10.0, None),
    ({"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": 0.0, "threshold": -2.0}, (-8, 5), -2.0, None),
    ({"unit": "mm/h", "transform": "log", "threshold": -1.5}, (-8, 5), -1.5, None),
    ({"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": 0.5, "threshold": -1.0}, (-1.99, 4), -1.0, 0.5),
    ({"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": 0.1, "threshold": -2.0}, (-9.99, 4), -2.0, 0.1),
    ({"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": 1e-3, "threshold": -2.0}, (-8, 5), -2.0, 1e-3),
    ({"unit": "mm/h", "transform": "BoxCox", "BoxCox_lambda": -0.5, "threshold": -1.0}, (-6, 1.99), -1.0, -0.5),
    ({"unit": "dBZ", "transform": None, "threshold": 0.1, "zerovalue": 0.0}, (0, 60), None, None),
    ({"unit": "dBZ", "transform": None, "threshold": 0.1, "zerovalue": 0.0, "zr_a": 316.0, "zr_b": 1.5}, (0, 60),
     None, None),
]


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("case", range(len(_CONVERSIONS)))
def test_conversion_within_bound_and_threshold_fixup(dt, case):
    meta, (lo, hi), thr, lam = _CONVERSIONS[case]
    rng = np.random.default_rng(case)
    x = rng.uniform(lo, hi, 200000).astype(dt)
    if lam is not None:  # arguments where lambda x + 1 -> 0
        x[100:200] = ((np.geomspace(1e-6, 1e-2, 100) - 1) / lam).astype(dt)
    near = 0
    if thr is not None:  # 2000 consecutive values around the threshold: the fix-up path
        it = np.int32 if dt == np.float32 else np.int64
        x[:2000] = (np.asarray(thr, dt).view(it) + np.arange(-1000, 1000, dtype=it)).view(dt)
        with np.errstate(all="ignore"):
            raw = ora.to_rainrate(x[:2000], dict(meta, threshold=-np.inf)).astype(np.float64)
            t = float(ora.to_rainrate(np.array([thr]), dict(meta, threshold=-np.inf))[0])
        eps = float(np.finfo(dt).eps)
        zz = np.abs(np.log(lam * x[:2000].astype(np.float64) + 1) / lam) if lam is not None else 0.0
        near = int((np.abs(raw - t) <= 8 * eps * (2 + zz) * np.maximum(np.abs(raw), t)).sum())
    got, fixed = _convert(x, meta)
    with np.errstate(all="ignore"):
        want = ora.to_rainrate(x, meta)
    assert got.dtype == want.dtype
    if thr is not None:
        # where NumPy's values come within half the bound of the threshold, the device lists pixels;
        # where they cannot (float32 Box-Cox with a tiny lambda steps by hundreds of ulp), it decides
        assert fixed >= 1 if near else True, (near, fixed)
        assert np.array_equal(got == 0, want == 0)  # NumPy's threshold decision, pixel for pixel
    ok = np.isfinite(want) & (want != 0)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    z = 0.0
    if lam is not None:
        with np.errstate(all="ignore"):
            z = np.abs(np.log(lam * x.astype(np.float64) + 1) / lam)[ok]
    err = np.abs(got[ok].astype(np.float64) - want[ok]) / np.spacing(want[ok]).astype(np.float64)
    assert np.all(err <= _bound_ulps(z)), float(err.max())


def test_numpy_and_tensor_input_agree_and_repeat():
    P, R = make_case(2, n_nwp=3, dt=np.float32)
    a = _run(P, R, True, True)
    b = _run(torch.from_numpy(P).cuda(), torch.from_numpy(R).cuda(), True, True)
    c = _run(P, R, True, True)
    assert isinstance(b, torch.Tensor) and b.is_cuda
    assert bits_equal(a, b.cpu().numpy()) and bits_equal(a, c)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 257, 4095, 4096, 4097, 12345, 70001])
def test_dense_rank_equals_unique(n):
    from pysteps_b200 import _device, _lib
    rng = np.random.default_rng(n)
    pool = np.array([0.0, -0.0, 5e-324, -5e-324, np.inf, -np.inf, 1.0, -1.0, 2.5e-310])
    for x in (rng.choice(pool, n), np.full(n, 3.0), rng.standard_normal(n), rng.standard_normal(n).astype(np.float32)):
        d = _device.to_device(np.ascontiguousarray(x))
        nb = _lib.c_i64(0)
        _lib.check(_lib.load().b200_blend_scratch_bytes(n, nb))
        scratch = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
        rank = torch.empty(n, dtype=torch.int32, device="cuda")
        info = torch.zeros(2, dtype=torch.int32, device="cuda")
        _lib.call("b200_dense_rank", d.data_ptr(), _device.dtype_code(d.dtype), n, rank.data_ptr(),
                  info[0:1].data_ptr(), info[1:2].data_ptr(), scratch.data_ptr(), nb.value, _device.stream_ptr())
        want = ora.dense_rank(x)
        assert np.array_equal(rank.cpu().numpy().astype(np.float64), want)
        assert int(info[0]) == int(want.max()) and int(info[1]) == 0


def test_dense_rank_large_slab():
    from pysteps_b200 import _device, _lib
    rng = np.random.default_rng(7)
    x = rng.gamma(0.5, 1.0, 24 * 1024 * 1024).astype(np.float32) - rng.gamma(0.5, 1.0, 24 * 1024 * 1024).astype(np.float32)
    n = x.size
    d = _device.to_device(x)
    nb = _lib.c_i64(0)
    _lib.check(_lib.load().b200_blend_scratch_bytes(n, nb))
    scratch = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    rank = torch.empty(n, dtype=torch.int32, device="cuda")
    info = torch.zeros(2, dtype=torch.int32, device="cuda")
    _lib.call("b200_dense_rank", d.data_ptr(), _device.dtype_code(d.dtype), n, rank.data_ptr(), info[0:1].data_ptr(),
              info[1:2].data_ptr(), scratch.data_ptr(), nb.value, _device.stream_ptr())
    assert np.array_equal(rank.cpu().numpy().astype(np.float64), ora.dense_rank(x))


def test_extrapolation_nowcast_equals_the_oracle():
    from oracle import semilagrangian as sl_ora
    from pysteps_b200.nowcasts import get_method
    rng = np.random.default_rng(3)
    P = rng.gamma(0.8, 2.0, (96, 112))
    P[rng.random(P.shape) < 0.02] = np.nan
    V = rng.uniform(-2, 2, (2, 96, 112))
    f = get_method("extrapolation")
    want = sl_ora.extrapolate(P, V, 5, allow_nonfinite_values=True)
    a = f(P, V, 5)
    b = f(torch.from_numpy(P).cuda(), torch.from_numpy(V).cuda(), 5)
    assert isinstance(a, np.ndarray) and isinstance(b, torch.Tensor) and b.is_cuda
    assert bits_equal(a, want) and bits_equal(b.cpu().numpy(), want)
    e = f(P, V, 3, extrap_method="eulerian")
    assert bits_equal(e, np.repeat(P[None], 3, axis=0))


def test_end_to_end_2048():
    """24 NWP members x 2048^2, T = 12 against the oracle fed the same nowcast: every lead and member
    on seeded pixel samples for the linear blend, and one whole lead of the salient blend."""
    from pysteps_b200.nowcasts import get_method
    rng = np.random.default_rng(0)
    m = 2048
    P = torch.from_numpy(rng.gamma(0.8, 2.0, (m, m))).cuda()
    R = torch.from_numpy(rng.gamma(0.8, 2.0, (24, 12, m, m)).astype(np.float32)).cuda()
    V = torch.from_numpy(rng.uniform(-3, 3, (2, m, m))).cuda()
    f = _ours().forecast
    kw = dict(start_blending=15, end_blending=45)
    meta = {"unit": "mm/h", "transform": None}
    now = get_method("extrapolation")(P, V, 9).cpu().numpy()
    Rh = R.cpu().numpy()
    pix = rng.integers(0, m * m, 4096)
    lin = f(P, meta, V, 12, 5, "extrapolation", R, meta, **kw)
    assert lin.shape == (24, 12, m, m) and lin.dtype == torch.float32
    want = ora.blend(now.reshape(9, -1)[:, pix, None], Rh.reshape(24, 12, -1)[:, :, pix, None], 12, 5, 15, 45)
    assert bits_equal(lin.reshape(24, 12, -1)[:, :, torch.from_numpy(pix).cuda()].cpu().numpy(), want[..., 0])
    del lin
    sal = f(P, meta, V, 12, 5, "extrapolation", R, meta, saliency=True, **kw)
    again = f(P, meta, V, 12, 5, "extrapolation", R, meta, saliency=True, **kw)
    assert torch.equal(sal, again)
    lead = 4  # t = 25: inside the window
    want = ora.blend(now[None, lead:lead + 1].repeat(24, axis=0), Rh[:, lead:lead + 1], 1, 25, 15, 45, True, True)
    assert bits_equal(sal[:, lead].cpu().numpy(), want[:, 0])
