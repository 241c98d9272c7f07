"""GPU parity tests of the semi-Lagrangian CUDA path (through the Python mirror ->
ctypes -> C ABI) against the CPU oracle and the committed reference outputs.
Bar: BIT-IDENTICAL outputs and displacements (trajectory arithmetic is float64 in
the reference's operation order; float32 outputs are the float64 value rounded once)."""
import ctypes

import numpy as np
import pytest
from conftest import assert_bits_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sl():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200.extrapolation import semilagrangian
    return semilagrangian


def _run_both(sl, args, kwargs):
    from oracle import semilagrangian as ora
    return sl.extrapolate(*args, **kwargs), ora.extrapolate(*args, **kwargs)


def _compare(got, want, name):
    if isinstance(want, tuple):
        assert isinstance(got, tuple)
        if want[0] is None:
            assert got[0] is None
        else:
            assert_bits_equal(got[0], want[0], name + " output")
        assert_bits_equal(got[1], want[1], name + " displacement")
    else:
        assert_bits_equal(got, want, name + " output")


def test_golden_cases(sl, golden_sl):
    from sl_cases import CASES, build_case
    for name in CASES:
        args, kwargs = build_case(name)
        res = sl.extrapolate(*args, **kwargs)
        if isinstance(res, tuple):
            out, disp = res
            assert_bits_equal(disp, golden_sl[name + "/disp"], name + " displacement")
        else:
            out = res
        if out is not None:
            assert_bits_equal(out, golden_sl[name + "/out"], name + " output")


def test_known_answers(sl):
    # pysteps/tests/test_extrapolation_semilagrangian.py:9-24 and :57-72
    precip = np.zeros((8, 8))
    precip[0, 0] = 1
    expected = np.zeros((8, 8))
    expected[:, 0] = np.nan
    expected[0, :] = np.nan
    expected[1, 1] = 1
    v = np.ones((8, 8))
    np.testing.assert_array_equal(sl.extrapolate(precip, np.stack([v, v]), 1)[0], expected)
    v = np.ones((8, 8)) * 10
    np.testing.assert_array_equal(sl.extrapolate(precip, np.stack([v, v]), [0.1])[0], expected)


def test_errors(sl):
    # pysteps/tests/test_extrapolation_semilagrangian.py:27-54 + semilagrangian.py:106-137
    v = np.ones((8, 8))
    V = np.stack([v, v])
    P = np.zeros((8, 8))
    with pytest.raises(ValueError, match="two-dimensional"):
        sl.extrapolate(np.zeros((8, 8, 8)), V, 1)
    with pytest.raises(ValueError, match="three-dimensional"):
        sl.extrapolate(P, v, 1)
    with pytest.raises(ValueError, match="ascending"):
        sl.extrapolate(P, V, [1, 0])
    with pytest.raises(ValueError, match="monotonously"):
        sl.extrapolate(P, V, [1, 1])
    Pn = P.copy()
    Pn[2, 2] = np.nan
    with pytest.raises(ValueError, match="precip contains non-finite"):
        sl.extrapolate(Pn, V, 1)
    Vn = V.copy()
    Vn[0, 1, 1] = np.inf
    with pytest.raises(ValueError, match="velocity contains non-finite"):
        sl.extrapolate(P, Vn, 1)
    with pytest.raises(ValueError, match="only non-finite"):
        sl.extrapolate(np.full((8, 8), np.nan), V, 1, allow_nonfinite_values=True)
    with pytest.raises(ValueError, match="velocity contains only"):
        sl.extrapolate(P, np.full((2, 8, 8), np.nan), 1, allow_nonfinite_values=True)
    with pytest.raises(ValueError, match="return_displacement is False"):
        sl.extrapolate(None, V, 1)
    with pytest.raises(RuntimeError, match="spline order not supported"):
        sl.extrapolate(P, V, 1, interp_order=6)
    with pytest.raises(NotImplementedError):
        sl.extrapolate(P, V, 1, map_coordinates_mode="wrap")
    with pytest.warns(UserWarning, match="D_prev"):
        sl.extrapolate(P, V, 1, D_prev=None)
    out = sl.extrapolate(P, V, 1, some_unknown_kwarg=5)  # unknown kwargs ignored (:29,129-134)
    assert out.shape == (1, 8, 8)
    # outval is only looked at when there is a field to warp (:171-172): "min" without precip is fine
    none, disp = sl.extrapolate(None, V, 2, "min", return_displacement=True)
    assert none is None and disp.shape == (2, 8, 8)


@pytest.mark.parametrize("shape,kind,T", [((257, 301), "smooth", 6), ((300, 200), "rotation", 12),
                                           ((64, 513), "smooth", 3), ((1, 50), "uniform", 2),
                                           ((50, 1), "uniform", 2), ((3, 3), "smooth", 2)])
def test_vs_oracle_shapes(sl, shape, kind, T):
    from pysteps_b200 import _synthetic as syn
    m, n = shape
    P = syn.rain_field(m, n, 2)
    V = syn.velocity_field(m, n, 2, kind) * (5.0 if kind == "rotation" else 1.0)
    got, want = _run_both(sl, (P, V, T), {"return_displacement": True})
    _compare(got, want, f"{shape} {kind}")


def test_vs_oracle_nonfinite_and_steps_call_shape(sl):
    """The call shape of nowcasts/utils.py:453-458 (single step, displacement carried)."""
    from pysteps_b200 import _synthetic as syn
    m, n = 200, 240
    P = syn.nan_disc(syn.rain_field(m, n, 4))
    V = syn.velocity_field(m, n, 4)
    x, y = np.meshgrid(np.arange(n), np.arange(m))
    xy = np.stack([x, y])
    disp_g = disp_o = None
    from oracle import semilagrangian as ora
    for step in range(3):
        kw = dict(allow_nonfinite_values=True, xy_coords=xy, return_displacement=True)
        g, disp_g = sl.extrapolate(P, V, [1.0], displacement_prev=disp_g, **kw)
        o, disp_o = ora.extrapolate(P, V, [1.0], displacement_prev=disp_o, **kw)
        assert_bits_equal(g, o, f"step {step} out")
        assert_bits_equal(disp_g, disp_o, f"step {step} disp")
    # carried single steps == one 3-step call (bitwise, property of the scheme)
    full, disp_full = sl.extrapolate(P, V, 3, allow_nonfinite_values=True, return_displacement=True)
    assert_bits_equal(g[0], full[2], "carried vs fused")
    assert_bits_equal(disp_g, disp_full, "carried vs fused disp")


def test_device_tensor_io(sl):
    import torch
    from pysteps_b200 import _synthetic as syn
    P = syn.rain_field(96, 128, 1).astype(np.float32)
    V = syn.velocity_field(96, 128, 1).astype(np.float32)
    host = sl.extrapolate(P, V, 4)
    dev = sl.extrapolate(torch.from_numpy(P).cuda(), torch.from_numpy(V).cuda(), 4)
    assert dev.is_cuda and dev.dtype == torch.float32
    assert_bits_equal(dev.cpu().numpy(), host, "device io")


def test_host_buffer_c_abi(sl):
    """b200_sl_extrapolate_host: the plain C entry point with host pointers."""
    from pysteps_b200 import _lib, _synthetic as syn
    from oracle import semilagrangian as ora
    lib = _lib.load()
    m, n, T = 120, 90, 5
    P = syn.rain_field(m, n, 6)
    V = syn.velocity_field(m, n, 6)
    out = np.empty((T, m, n))
    disp = np.empty((2, m, n))
    td = np.ones(T)
    vp = ctypes.c_void_p
    rc = lib.b200_sl_extrapolate_host(P.ctypes.data_as(vp), V.ctypes.data_as(vp), None, None,
                                      td.ctypes.data_as(_lib.c_dp), T, 1.0, 1, float("nan"),
                                      _lib.MODE_CONSTANT, _lib.F64, _lib.F64, m, n,
                                      out.ctypes.data_as(vp), disp.ctypes.data_as(vp))
    _lib.check(rc)
    want, wdisp = ora.extrapolate(P, V, T, return_displacement=True)
    assert_bits_equal(out, want, "host abi out")
    assert_bits_equal(disp, wdisp, "host abi disp")
    rc = lib.b200_sl_extrapolate_host(None, None, None, None, td.ctypes.data_as(_lib.c_dp), T, 1.0,
                                      1, 0.0, 0, _lib.F64, _lib.F64, m, n, None, None)
    assert rc != 0 and b"bad arguments" in lib.b200_last_error()


def test_full_size_properties(sl):
    """BASELINE.json size (2048^2, 12 leadtimes): size-independent properties."""
    import torch
    from pysteps_b200 import _synthetic as syn
    m = n = 2048
    P = syn.rain_field(m, n, 0).astype(np.float32)
    dP = torch.from_numpy(P).cuda()
    # zero motion: identity at every leadtime
    out = sl.extrapolate(dP, torch.zeros((2, m, n), device="cuda"), 12)
    assert bool((out == dP[None]).all())
    # uniform integer motion: exact translation with NaN inflow
    V = torch.zeros((2, m, n), device="cuda")
    V[0] = 3.0
    V[1] = -2.0
    out = sl.extrapolate(dP, V, 12)
    for t in (0, 5, 11):
        k = t + 1
        ref = np.full((m, n), np.nan, dtype=np.float32)
        ref[: m - 2 * k, 3 * k:] = P[2 * k:, : n - 3 * k]
        assert_bits_equal(out[t].cpu().numpy(), ref, f"translation t={t}")
    # fused 12 leadtimes == 12 carried single steps, bitwise; and the whole result against the oracle
    from oracle import semilagrangian as ora
    Vh = syn.velocity_field(m, n, 0, "rotation").astype(np.float32)
    Vs = torch.from_numpy(Vh).cuda()
    full, dfull = sl.extrapolate(dP, Vs, 12, return_displacement=True)
    d = None
    for t in range(12):
        o, d = sl.extrapolate(dP, Vs, [1.0], displacement_prev=d, return_displacement=True)
        assert torch.equal(torch.nan_to_num(o[0], nan=-1.0), torch.nan_to_num(full[t], nan=-1.0))
    assert torch.equal(d, dfull)
    want, wdisp = ora.extrapolate(P, Vh, 12, return_displacement=True)
    assert_bits_equal(full.cpu().numpy(), want, "full size vs oracle")
    assert_bits_equal(dfull.cpu().numpy(), wdisp, "full size displacement vs oracle")


def test_row_bands_equal_full_frame(sl):
    """Tile partitioning (config[4]): any output band computed alone is bitwise the
    corresponding rows of the full-frame result, incl. carried displacements."""
    from pysteps_b200 import _shard, _synthetic as syn
    m, n = 301, 260
    P = syn.nan_disc(syn.rain_field(m, n, 9))
    V = syn.velocity_field(m, n, 9, "rotation") * 6.0
    full, dfull = sl.extrapolate(P, V, 5, allow_nonfinite_values=True, return_displacement=True)
    covered = 0
    for rank in range(3):
        r0, r1 = _shard.row_band(m, 3, rank)
        band, dband = sl.extrapolate(P, V, 3, allow_nonfinite_values=True, return_displacement=True,
                                     b200_rows=(r0, r1))
        band2, dband2 = sl.extrapolate(P, V, [1.0, 2.0], allow_nonfinite_values=True,
                                       return_displacement=True, displacement_prev=dband, b200_rows=(r0, r1))
        assert band.shape == (3, r1 - r0, n)
        assert_bits_equal(band, full[:3, r0:r1], f"band {rank}")
        assert_bits_equal(band2, full[3:, r0:r1], f"band {rank} continued")
        assert_bits_equal(dband2, dfull[:, r0:r1], f"band {rank} displacement")
        covered += r1 - r0
    assert covered == m


def test_concurrent_calls_from_threads(sl):
    """nowcasts/utils.py:464-468 calls the extrapolator from dask threads: concurrent calls must
    not interfere (stream-ordered scratch, no global mutable state in the kernels)."""
    from concurrent.futures import ThreadPoolExecutor
    from pysteps_b200 import _synthetic as syn
    cases = []
    for i in range(6):
        P = syn.rain_field(180 + 8 * i, 200, 20 + i)
        V = syn.velocity_field(180 + 8 * i, 200, 20 + i, "rotation") * (2.0 + i)
        cases.append((P, V))
    serial = [sl.extrapolate(P, V, 4, return_displacement=True) for P, V in cases]
    with ThreadPoolExecutor(max_workers=6) as ex:
        futs = [ex.submit(sl.extrapolate, P, V, 4, return_displacement=True) for P, V in cases for _ in range(3)]
        res = [f.result() for f in futs]
    for k, (out, disp) in enumerate(res):
        assert_bits_equal(out, serial[k // 3][0], f"thread result {k}")
        assert_bits_equal(disp, serial[k // 3][1], f"thread displacement {k}")


def test_randomised_differential_vs_oracle(sl):
    """40 random argument combinations (shapes incl. degenerate axes, dtypes, n_iter, integer /
    list timesteps, modes, outval, carried displacement, custom coordinates, NaNs): outputs and
    displacements bit-identical to the oracle every time."""
    from oracle import semilagrangian as ora
    rng = np.random.default_rng(2024)
    for trial in range(40):
        m = int(rng.choice([1, 2, 3, 17, 64, 97, 130]))
        n = int(rng.choice([1, 2, 5, 33, 64, 101, 257]))
        pdt = rng.choice([np.float32, np.float64])
        vdt = rng.choice([np.float32, np.float64])
        P = (rng.gamma(1.0, 4.0, (m, n)) * (rng.random((m, n)) > 0.5)).astype(pdt)
        V = (rng.normal(size=(2, m, n)) * rng.choice([0.3, 2.0, 9.0]) + rng.normal(size=(2, 1, 1))).astype(vdt)
        kw = {}
        if rng.random() < 0.3:
            P = P.copy()
            P[rng.integers(0, m), rng.integers(0, n)] = np.nan
            if m * n > 1:
                kw["allow_nonfinite_values"] = True
            else:
                P = np.nan_to_num(P)
        kw["n_iter"] = int(rng.choice([0, 1, 1, 1, 2, 3]))
        if rng.random() < 0.5:
            ts = int(rng.integers(1, 5))
        else:
            ts = sorted(set(np.round(rng.uniform(0.1, 4.0, int(rng.integers(1, 4))), 3).tolist()))
            kw["vel_timestep"] = float(rng.choice([1.0, 2.0, 5.0]))
        kw["map_coordinates_mode"] = str(rng.choice(["constant", "nearest"]))
        outval = rng.choice(["nan", "min", "num"])
        outval = {"nan": np.nan, "min": "min", "num": -3.25}[outval]
        if rng.random() < 0.5:
            kw["return_displacement"] = True
        if rng.random() < 0.35:
            kw["displacement_prev"] = rng.normal(size=(2, m, n)) * 3.0
        if rng.random() < 0.25:
            x, y = np.meshgrid(np.arange(n) * 0.9 + 0.3, np.arange(m) * 1.1 - 0.2)
            kw["xy_coords"] = np.stack([x, y])
        got = sl.extrapolate(P, V, ts, outval, **kw)
        want = ora.extrapolate(P, V, ts, outval, **kw)
        _compare(got, want, f"trial {trial}: {(m, n)} {pdt.__name__}/{vdt.__name__} ts={ts} {sorted(kw)}")


# ---------------------------------------------------------------------------------------------
# opt-in float32-tap kernel (b200_float32_taps=True): tolerance on values, certified tap indices
F32_VALUE_TOL = 2e-5     # |out - exact| <= F32_VALUE_TOL * max|precip| (finite pixels)
F32_DISP_TOL = 1e-4      # |displacement - exact| in pixels (measured: 2e-6 smooth field, 3e-5 at |V| ~ 50 px/step)


@pytest.mark.parametrize("kind,scale,pdtype", [("smooth", 1.0, np.float32), ("rotation", 4.0, np.float64),
                                               ("smooth", 0.0, np.float32), ("rotation", 12.0, np.float32)])
def test_float32_taps_indices_and_tolerance(sl, kind, scale, pdtype):
    """Every leadtime's end-point coordinates floor to the SAME tap indices as the exact kernel (the
    displacement after k leadtimes is the k-th end-point sample), values and displacements inside the
    stated float32 tolerance, NaN pattern identical."""
    import torch
    from pysteps_b200 import _synthetic as syn
    m, n = 384, 448
    P = syn.rain_field(m, n, 3).astype(pdtype)
    V = syn.velocity_field(m, n, 3, kind) * scale
    yy, xx = np.meshgrid(np.arange(m, dtype=np.float64), np.arange(n, dtype=np.float64), indexing="ij")
    pmax = float(np.abs(P).max())
    for T in (1, 2, 5, 12):
        exact, dex = sl.extrapolate(P, V, T, return_displacement=True)
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        fast, dfa = sl.extrapolate(P, V, T, return_displacement=True, b200_float32_taps=True,
                                   b200_fallback_count=cnt)
        assert fast.dtype == exact.dtype and fast.shape == exact.shape
        assert np.array_equal(np.isnan(fast), np.isnan(exact)), "NaN pattern"
        ok = ~np.isnan(exact)
        err = np.abs(fast[ok].astype(np.float64) - exact[ok].astype(np.float64)).max() if ok.any() else 0.0
        assert err <= F32_VALUE_TOL * pmax, f"T={T}: value error {err:.3e} (max|P| {pmax:.3g})"
        assert np.abs(dfa - dex).max() <= F32_DISP_TOL, f"T={T}: displacement error {np.abs(dfa - dex).max():.3e}"
        # integer tap indices of the last end-point sample: identical at EVERY pixel
        assert np.array_equal(np.floor(xx + dfa[0]), np.floor(xx + dex[0])), f"T={T}: column indices"
        assert np.array_equal(np.floor(yy + dfa[1]), np.floor(yy + dex[1])), f"T={T}: row indices"
        frac = int(cnt.item()) / (m * n)
        if scale > 0 and kind == "smooth":
            assert frac < 0.2, f"T={T}: {frac:.3f} of the pixels fell back to the exact code"
    # zero motion: every sample sits ON a cell boundary -> all pixels take the exact path -> identity
    if scale == 0.0:
        assert_bits_equal(fast, exact, "zero motion")


def test_float32_taps_modes_nonfinite_bands_and_carry(sl):
    """mode / outval / NaN rules are the exact kernel's (uncertified pixels ARE the exact kernel); the
    STEPS call shape (single steps with carried displacement) and row bands work as in the exact path."""
    from pysteps_b200 import _shard, _synthetic as syn
    m, n = 200, 240
    P = syn.nan_disc(syn.rain_field(m, n, 4))
    V = syn.velocity_field(m, n, 4, "rotation") * 5.0
    pmax = float(np.nanmax(np.abs(P)))
    for kw in (dict(allow_nonfinite_values=True), dict(allow_nonfinite_values=True, outval=0.0),
               dict(allow_nonfinite_values=True, map_coordinates_mode="nearest")):
        exact, dex = sl.extrapolate(P, V, 6, return_displacement=True, **kw)
        fast, dfa = sl.extrapolate(P, V, 6, return_displacement=True, b200_float32_taps=True, **kw)
        assert np.array_equal(np.isnan(fast), np.isnan(exact)), f"NaN pattern {kw}"
        ok = ~np.isnan(exact)
        assert np.abs(fast[ok] - exact[ok]).max() <= F32_VALUE_TOL * pmax
        assert np.abs(dfa - dex).max() <= F32_DISP_TOL
    # carried single steps
    kw = dict(allow_nonfinite_values=True, return_displacement=True)
    full, dfull = sl.extrapolate(P, V, 4, **kw)
    d = None
    for t in range(4):
        o, d = sl.extrapolate(P, V, [1.0], displacement_prev=d, b200_float32_taps=True, **kw)
        ok = ~np.isnan(full[t])
        assert np.array_equal(np.isnan(o[0]), np.isnan(full[t]))
        assert np.abs(o[0][ok] - full[t][ok]).max() <= F32_VALUE_TOL * pmax
    assert np.abs(d - dfull).max() <= F32_DISP_TOL
    # a band alone == the rows of the full float32-tap frame, bitwise (same kernel, same pixels)
    fast, dfa = sl.extrapolate(P, V, 3, b200_float32_taps=True, **kw)
    r0, r1 = _shard.row_band(m, 3, 1)
    band, dband = sl.extrapolate(P, V, 3, b200_float32_taps=True, b200_rows=(r0, r1), **kw)
    assert_bits_equal(band, fast[:, r0:r1], "band")
    assert_bits_equal(dband, dfa[:, r0:r1], "band displacement")
    # what the variant does not cover is refused, not silently computed otherwise
    with pytest.raises(NotImplementedError):
        sl.extrapolate(P, V, 2, allow_nonfinite_values=True, b200_float32_taps=True, n_iter=3)
    with pytest.raises(NotImplementedError):
        sl.extrapolate(P, V, 2, allow_nonfinite_values=True, b200_float32_taps=True, interp_order=3)


def test_float32_taps_full_size(sl):
    """BASELINE size: tolerance, indices and the share of recomputed pixels on the LK-like smooth field."""
    import torch
    from pysteps_b200 import _synthetic as syn
    m = n = 2048
    P = torch.from_numpy(syn.rain_field(m, n, 0).astype(np.float32)).cuda()
    V = torch.from_numpy(syn.velocity_field(m, n, 0, "smooth")).cuda()
    exact, dex = sl.extrapolate(P, V, 12, return_displacement=True)
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    fast, dfa = sl.extrapolate(P, V, 12, return_displacement=True, b200_float32_taps=True, b200_fallback_count=cnt)
    assert torch.equal(torch.isnan(fast), torch.isnan(exact))
    err = torch.nan_to_num((fast.double() - exact.double()).abs(), nan=0.0).max().item()
    assert err <= F32_VALUE_TOL * float(P.abs().max()), f"value error {err:.3e}"
    assert (dfa - dex).abs().max().item() <= F32_DISP_TOL
    gy, gx = torch.meshgrid(torch.arange(m, device="cuda", dtype=torch.float64),
                            torch.arange(n, device="cuda", dtype=torch.float64), indexing="ij")
    assert torch.equal(torch.floor(gx + dfa[0]), torch.floor(gx + dex[0]))
    assert torch.equal(torch.floor(gy + dfa[1]), torch.floor(gy + dex[1]))
    frac = cnt.item() / (m * n)
    print(f"float32 taps 2048^2 T=12: max value error {err:.3e}, max displacement error "
          f"{(dfa - dex).abs().max().item():.3e}, {100 * frac:.3f} % of the pixels recomputed exactly")
    assert frac < 0.05


@pytest.mark.parametrize("mag", [3.0e9, 5.0e9, 1.0e19, 2147483648.5])
def test_absurd_displacements_follow_the_reference(sl, mag):
    """Coordinates of 2^31 pixels and beyond: the interior test reads the floor from the low word of a
    magic-constant sum, so an index >= 2^31 must not pass as a small negative one.  (The reference goes
    through `(npy_intp)floor(c)`; the oracle reproduces it, incl. the INT64_MIN of out-of-range values.)"""
    from pysteps_b200 import _synthetic as syn
    m, n = 40, 56
    P = syn.rain_field(m, n, 8) + 1.0
    V = np.zeros((2, m, n))
    V[0, :, ::2] = -mag      # backward trajectory: coordinates x + mag (columns), rows untouched
    V[1, ::3, :] = mag       # coordinates y - mag
    V[0, 5:9, 5:9] = 1.5     # and ordinary pixels among them
    for kw in (dict(), dict(map_coordinates_mode="nearest"), dict(outval=-1.0, n_iter=2)):
        got, want = _run_both(sl, (P, V, 2), dict(return_displacement=True, **kw))
        _compare(got, want, f"|V| = {mag:g} {kw}")
