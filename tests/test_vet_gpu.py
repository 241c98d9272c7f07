"""GPU parity tests of the VET CUDA path (csrc/vet.cu behind pysteps_b200.motion.vet)
against the CPU oracle and the committed reference outputs.  Bars: single cost / gradient
evaluations relative 1e-12 (same float64 operations, different summation tree); morphing and
zoom bit-identical; optimised fields 1e-6 px vs oracle and reference; repeated evaluations
bit-identical run to run (pysteps/tests/test_motion.py:381-396 asks 1e-12)."""
import os

import numpy as np
import pytest
from conftest import assert_bits_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vet():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200.motion import vet as v
    return v


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "vet_golden.npz"))


def test_cost_and_gradient(vet, golden):
    from oracle import vet as ora
    from vet_cases import EVAL_CASES, eval_case
    for name in EVAL_CASES:
        sd, images, mask, gain = eval_case(name)
        shape = sd.shape[1:]
        c = vet.vet_cost_function(sd.ravel(), images, shape, mask, gain)
        g = vet.vet_cost_function_gradient(sd.ravel(), images, shape, mask, gain)
        co = ora.vet_cost_function(sd.ravel(), images, shape, mask, gain)
        go = ora.vet_cost_function_gradient(sd.ravel(), images, shape, mask, gain)
        assert abs(c - co) <= 1e-12 * abs(co), name
        assert np.abs(g - go).max() <= 1e-12 * np.abs(go).max(), name
        assert abs(c - golden[name + "/cost"]) <= 1e-9 * abs(golden[name + "/cost"])
        assert np.abs(g - golden[name + "/grad"]).max() <= 1e-9 * np.abs(golden[name + "/grad"]).max()
        # smooth_gain = 0 switches the smoothness term off
        c0 = vet.vet_cost_function(sd.ravel(), images, shape, mask, 0.0)
        assert abs(c0 - ora.vet_cost_function(sd.ravel(), images, shape, mask, 0.0)) <= 1e-12 * abs(c0)


def test_repeatability(vet):
    from vet_cases import eval_case
    sd, images, mask, gain = eval_case("eval_256x256_s32x32")
    shape = sd.shape[1:]
    c0 = vet.vet_cost_function(sd.ravel(), images, shape, mask, gain)
    g0 = vet.vet_cost_function_gradient(sd.ravel(), images, shape, mask, gain)
    for _ in range(20):
        assert vet.vet_cost_function(sd.ravel(), images, shape, mask, gain) == c0
        assert np.array_equal(vet.vet_cost_function_gradient(sd.ravel(), images, shape, mask, gain), g0)


def test_morph_and_zoom(vet, golden):
    import torch
    from oracle import vet as ora
    from pysteps_b200 import _lib
    from vet_cases import eval_case
    img = eval_case("eval_128x160_s4x4")[1][0]
    w, wm, wg = vet.morph(img, golden["morph/disp"], gradient=True)
    ow, owm, owg = ora.warp(img, np.zeros(img.shape, np.int8), golden["morph/disp"], gradient=True)
    assert_bits_equal(w, ow, "morphed image")
    assert np.array_equal(wm, owm)
    assert_bits_equal(wg, owg, "morph gradient")
    assert np.abs(w - golden["morph/image"]).max() < 1e-12 and np.array_equal(wm, golden["morph/mask"])
    w2, wm2 = vet.morph(np.ma.masked_where(img > 20, img), golden["morph/disp"])
    o2, om2 = ora.warp(img, (img > 20).astype(np.int8), golden["morph/disp"])
    assert_bits_equal(w2, o2, "masked morph")
    assert np.array_equal(wm2, om2), "masked morph mask"
    rng = np.random.default_rng(0)
    for (c, h, w_, oh, ow_) in [(2, 2, 2, 4, 4), (2, 16, 16, 32, 32), (2, 3, 5, 7, 64), (2, 32, 32, 2048, 2048),
                                (2, 32, 16, 504, 1016)]:
        a = rng.normal(size=(c, h, w_))
        da = torch.from_numpy(a).cuda()
        out = torch.empty((c, oh, ow_), dtype=torch.float64, device="cuda")
        _lib.call("b200_zoom_bilinear", da.data_ptr(), c, h, w_, oh, ow_, out.data_ptr(),
                  torch.cuda.current_stream().cuda_stream)
        assert_bits_equal(out.cpu().numpy(), ora.zoom_o1(a, oh, ow_), f"zoom {(c, h, w_, oh, ow_)}")


def test_fused_pair_equals_separate_evaluations(vet):
    """b200_vet_value_and_gradient (one pass, value + gradient) is bitwise b200_vet_cost's value and
    b200_vet_cost's gradient, two and three frames (pairs summed in vet.py:257-293's order)."""
    import torch
    from pysteps_b200 import _lib
    from vet_cases import EVAL_CASES, eval_case
    s = torch.cuda.current_stream().cuda_stream
    for name in EVAL_CASES:
        sd, images, mask, gain = eval_case(name)
        T, nx, ny = images.shape
        _, xs, ys = sd.shape
        d_im, d_mk, d_sd = torch.from_numpy(images).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(sd).cuda()
        pairs = ((1, 2), (0, 1)) if T == 3 else ((0, 1),)
        res = smo = grad = None
        for a, b in pairs:
            oc = torch.empty(2, dtype=torch.float64, device="cuda")
            og = torch.empty((2, xs, ys), dtype=torch.float64, device="cuda")
            for mode, out in ((0, oc), (1, og)):
                _lib.call("b200_vet_cost", d_sd.data_ptr(), d_im[a].data_ptr(), d_im[b].data_ptr(), d_mk.data_ptr(),
                          xs, ys, nx, ny, gain, mode, out.data_ptr(), s)
            c, g = oc.cpu().numpy(), og.cpu().numpy()
            res, smo, grad = (c[0], c[1], g) if res is None else (res + c[0], smo + c[1], grad + g)
        work = torch.empty(3 * sd.size + 4, dtype=torch.float64, device="cuda")
        val, gout = np.zeros(2), np.zeros(sd.size)
        _lib.call("b200_vet_value_and_gradient", sd.ctypes.data, d_im.data_ptr(), T, d_mk.data_ptr(), xs, ys, nx, ny,
                  gain, work.data_ptr(), val.ctypes.data, gout.ctypes.data, s)
        assert val[0] == res and val[1] == smo, name
        assert np.array_equal(gout.reshape(2, xs, ys), grad), name


def test_level_images_kernel_equals_numpy_pad(vet):
    """b200_vet_level_images against vet.py:500-523 / :548-561 spelled with numpy.pad."""
    import torch
    from pysteps_b200 import _lib
    rng = np.random.default_rng(5)
    s = torch.cuda.current_stream().cuda_stream
    for T, m, n, gpad, (pi0, pi1), (pj0, pj1), masked in ((2, 37, 41, 0, (0, 0), (0, 0), False),
                                                         (3, 50, 33, 0, (3, 4), (1, 2), False),
                                                         (2, 29, 64, 5, (2, 3), (0, 0), False),
                                                         (3, 31, 45, 2, (1, 1), (7, 8), True)):
        fr = rng.standard_normal((T, m, n))
        fr[rng.random((T, m, n)) < 0.05] = np.nan
        fr[0, 3, 4] = np.inf
        um = rng.random((T, m, n)) < 0.1
        bad = um if masked else ~np.isfinite(fr)
        ref, rbad = fr.copy(), bad.copy()
        if gpad:
            tup = ((0, 0), (gpad, gpad), (gpad, gpad))
            ref = np.pad(ref, tup, "constant", constant_values=np.nan)
            rbad = np.pad(rbad, tup, "constant", constant_values=True)
        ref[rbad] = 0
        want = np.pad(ref, ((0, 0), (pi0, pi1), (pj0, pj1)), "edge")
        wmask = np.pad(np.any(rbad, axis=0).astype(np.int8), ((pi0, pi1), (pj0, pj1)), "constant", constant_values=1)
        M, N = want.shape[1:]
        d_fr = torch.from_numpy(fr).cuda()
        d_um = torch.from_numpy(um.astype(np.uint8)).cuda() if masked else None
        out = torch.empty((T, M, N), dtype=torch.float64, device="cuda")
        omask = torch.empty((M, N), dtype=torch.int8, device="cuda")
        _lib.call("b200_vet_level_images", d_fr.data_ptr(), None if d_um is None else d_um.data_ptr(), T, m, n,
                  gpad, pi0, pj0, M, N, out.data_ptr(), omask.data_ptr(), s)
        from conftest import assert_bits_equal
        assert_bits_equal(out.cpu().numpy(), want, "level images")
        assert np.array_equal(omask.cpu().numpy(), wmask)


def test_optimised_fields(vet, golden):
    from oracle import vet as ora
    from vet_cases import FIELD_CASES, field_case
    for name in FIELD_CASES:
        images, kw = field_case(name)
        field, steps = vet.vet(images, verbose=False, intermediate_steps=True, **kw)
        ofield = ora.vet(images, verbose=False, **kw)
        assert field.shape == ofield.shape and field.dtype == np.float64
        assert np.abs(field - ofield).max() < 1e-6, name
        assert np.abs(field - golden[name + "/field"]).max() < 1e-6, name
        for k, s in enumerate(steps):
            assert np.abs(s - golden[name + f"/step{k}"]).max() < 1e-6


def test_api_behaviour(vet):
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200.motion import get_method
    assert get_method("VET") is vet.vet
    fr = syn.rain_frames(96, 96, 2, 4)
    with pytest.raises(ValueError, match="dimension mismatch"):
        vet.vet(fr[0], verbose=False)
    with pytest.raises(ValueError, match="frames"):
        vet.vet(np.zeros((4, 32, 32)), verbose=False)
    with pytest.raises(ValueError, match="indexing"):
        vet.vet(fr, verbose=False, indexing="zz")
    with pytest.raises(ValueError, match="initial guess"):
        vet.vet(fr, verbose=False, first_guess=np.zeros((2, 3, 3)))
    # output shape preserved for prime-sized inputs and paddings (tests/test_motion.py:331-362)
    for shape, pad in (((101, 103), 0), ((101, 103), 3), ((97, 89), 10)):
        out = vet.vet(syn.rain_frames(shape[0], shape[1], 2, 1), verbose=False, padding=pad,
                      sectors=((8, 4, 2), (8, 4, 2)))
        assert out.shape == (2,) + shape
    # ndarray-with-NaN == MaskedArray input (tests/test_motion.py:400-430)
    frn = fr.copy()
    frn[:, 20:40, 30:50] = np.nan
    a = vet.vet(frn, verbose=False, sectors=((8, 4, 2), (8, 4, 2)))
    b = vet.vet(np.ma.masked_invalid(frn), verbose=False, sectors=((8, 4, 2), (8, 4, 2)))
    assert np.array_equal(a, b)
    # no precipitation -> ~zero motion (tests/test_motion.py:265-289: |uv| < 0.01)
    assert np.abs(vet.vet(np.zeros((2, 64, 64)), verbose=False)).max() < 0.01
    # recovers a translation; "yx" flips components to (u, v) (vet.py:639-640)
    V = vet.vet(syn.rain_frames(256, 256, 2, 3), verbose=False)
    wet = syn.rain_frames(256, 256, 2, 3)[1] > 0
    assert abs(V[0][wet].mean() - 3.0) < 0.1 and abs(V[1][wet].mean() + 2.0) < 0.1
