"""GPU tests of the VET kernels (csrc/vet.cu) on the edge grid of tests/vet_edges.py:
  - single-pixel probes through b200_vet_cost (modes 0 and 1): the residual bit for bit and every gradient
    component bit for bit (signed zeros equal) against the NumPy restatement and, on the small geometries,
    the C oracle; with a smoothness gain the residual bit for bit and the rest within its bound;
  - whole fields: every output within gamma_D * sum |term| of the exact sum, D the deepest addition chain
    of the launch's partition, and within the sum of both bounds of the oracle; three frames and the
    float smoothness gain through b200_vet_value_and_gradient and the public vet_cost_function*;
  - b200_vet_value_and_gradient bitwise equal to separate mode-0 and mode-1 calls on every geometry;
  - b200_vet_warp bit for bit against the oracle's warp on clamping, integer and exact-last-row
    displacements, and b200_zoom_bilinear at one output row or column.
The strip regimes are asserted on the SM count of the device at hand."""
import numpy as np
import pytest
from conftest import assert_bits_equal

import vet_edges as E
from oracle import vet as ora

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _lib, torch.cuda.get_device_properties(0).multi_processor_count


def _stream(torch):
    return torch.cuda.current_stream().cuda_stream


def _dev_cost(env, sd, templ, inp, mask, gain):
    """b200_vet_cost in modes 0 and 1 -> (residual, smoothness, gradient (2, xs, ys))"""
    torch, L, _ = env
    nx, ny = templ.shape
    _, xs, ys = sd.shape
    d = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (sd, templ, inp, mask)]
    oc = torch.full((2,), -7.0, dtype=torch.float64, device="cuda")
    og = torch.full((2, xs, ys), -7.0, dtype=torch.float64, device="cuda")
    for mode, out in ((0, oc), (1, og)):
        L.call("b200_vet_cost", d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), xs, ys, nx, ny,
               gain, mode, out.data_ptr(), _stream(torch))
    c = oc.cpu().numpy()
    return c[0], c[1], og.cpu().numpy()


def _dev_pair(env, sd, images, mask, gain):
    """b200_vet_value_and_gradient -> ((residuals, smoothness), gradient (2, xs, ys))"""
    torch, L, _ = env
    T, nx, ny = images.shape
    _, xs, ys = sd.shape
    d_im, d_mk = torch.from_numpy(images).cuda(), torch.from_numpy(mask).cuda()
    work = torch.empty(3 * sd.size + 4, dtype=torch.float64, device="cuda")
    val, grad = np.zeros(2), np.zeros(sd.size)
    L.call("b200_vet_value_and_gradient", sd.ctypes.data, d_im.data_ptr(), T, d_mk.data_ptr(), xs, ys, nx, ny, gain,
           work.data_ptr(), val.ctypes.data, grad.ctypes.data, _stream(torch))
    return val, grad.reshape(2, xs, ys)


def _bits(a):
    return np.float64(a).view(np.int64)


def test_strip_regimes_on_this_device(env):
    _, _, sms = env
    reached = set()
    for nx, ny, xs, ys in E.GEOMETRIES.values():
        reached |= E.partition(nx, ny, xs, ys, sms)["regimes"]
    assert reached >= E.REGIMES, f"{sms} SMs: {sorted(E.REGIMES - reached)} not reached"
    print(f"{sms} SMs: bench levels in {[E.partition(*E.GEOMETRIES[g], sms)['strips'] for g in E.BENCH]} strips")


@pytest.mark.parametrize("geo", list(E.GEOMETRIES))
def test_probes_bit_for_bit(env, geo):
    _, _, sms = env
    small = geo not in E.BENCH
    pts = E.probe_points(geo, sms, small)
    got = E.probe_branches(geo, pts, sms)
    p = E.partition(*E.GEOMETRIES[geo], sms)
    assert "skipped row" in got and ("last strip first row" in got or max(p["used"]) == 1)
    for k, pt in enumerate(pts):
        sd, templ, inp, mask = E.probe_case(geo, pt)
        res, grad, _ = E.probe_expect(geo, pt, sd, templ, inp, mask)
        r, s, g = _dev_cost(env, sd, templ, inp, mask, 0.0)
        assert _bits(r) == _bits(res), (geo, pt, r, res)
        assert s == 0.0
        bad = np.argwhere(g != grad)
        assert bad.size == 0, (geo, pt, "gradient differs at", bad[:4].tolist(), g[tuple(bad[0])], grad[tuple(bad[0])])
        if small:
            ro = ora.cost_function(sd, templ, inp, mask, 0.0)[0]
            go = ora.cost_function(sd, templ, inp, mask, 0.0, gradient=True)
            assert _bits(ro) == _bits(r) and np.array_equal(go, g), (geo, pt)
        if small or k % 4 == 0:
            # with the smoothness term: the residual bit for bit, penalty and gradient within their bounds
            ev = E.probe_eval(geo, pt, sd, templ, inp, mask, 1e6)
            r, s, g = _dev_cost(env, sd, templ, inp, mask, 1e6)
            assert _bits(r) == _bits(res), (geo, pt)
            ch = E.chains(p)
            E.check_sums(r, s, g, ev, (ch["res"], ch["smooth"], ch["grad"]))


def _field(name):
    sd, images, mask, gain, geo = E.field_case(name)
    pairs = ((1, 2), (0, 1)) if len(images) == 3 else ((0, 1),)
    evs = [E.evaluate(sd, images[a], images[b], mask, gain) for a, b in pairs]
    return sd, images, mask, gain, geo, pairs, evs


@pytest.mark.parametrize("name", list(E.FIELD_CASES))
def test_fields_within_bound_of_exact_and_oracle(env, name):
    _, _, sms = env
    sd, images, mask, gain, geo, pairs, evs = _field(name)
    p = E.partition(*E.GEOMETRIES[geo], sms)
    ch = E.chains(p)
    Ddev = (ch["res"], ch["smooth"], ch["grad"])
    for (a, b), ev in zip(pairs, evs):
        r, s, g = _dev_cost(env, sd, images[a], images[b], mask, gain)
        E.check_sums(r, s, g, ev, Ddev)
        if E.FIELD_CASES[name][2] == "all":
            assert r == 0.0
        # the oracle: within both bounds of the same exact sums
        ro, so = ora.cost_function(sd, images[a], images[b], mask, gain)
        go = ora.cost_function(sd, images[a], images[b], mask, gain, gradient=True)
        Dora = E.oracle_chains(ev)
        tol_r = E.gamma(Ddev[0] + E.SLACK) * ev["res_abs"] + E.gamma(Dora[0] + E.SLACK) * ev["res_abs"]
        assert abs(r - ro) <= tol_r, (name, r, ro)
        tol_g = (E.gamma(Ddev[2] + E.SLACK) + E.gamma(Dora[2] + E.SLACK)) * ev["grad_abs"] + \
            2 * E.gamma(12 + E.SLACK) * ev["sgrad_abs"]
        assert (np.abs(g - go) <= tol_g).all(), (name, np.argwhere(np.abs(g - go) > tol_g)[:4].tolist())
    # the evaluation as the optimiser asks for it: one fused call over all pairs, pairs summed on the host
    ev = evs[0] if len(evs) == 1 else E.add_pairs(*evs)
    ch = E.chains(p, len(images))
    (r, s), g = _dev_pair(env, sd, images, mask, gain)
    E.check_sums(r, s, g, ev, (ch["res"], ch["smooth"], ch["grad"]))


@pytest.mark.parametrize("name", [n for n, c in E.FIELD_CASES.items() if c[0] not in E.BENCH])
def test_public_wrapper_rounds_the_gain_to_float(env, name):
    """vet_cost_function(_gradient) with the gain as given (0.1 is rounded to a float on the way in): the
    value is residuals + penalty, one more addition"""
    from pysteps_b200.motion import vet
    sd, images, mask, gain, geo, pairs, evs = _field(name)
    ev = evs[0] if len(evs) == 1 else E.add_pairs(*evs)
    ch = E.chains(E.partition(*E.GEOMETRIES[geo], env[2]), len(images))
    shape = sd.shape[1:]
    c = vet.vet_cost_function(sd.ravel(), images, shape, mask, gain)
    g = vet.vet_cost_function_gradient(sd.ravel(), images, shape, mask, gain).reshape(sd.shape)
    D = max(ch["res"], ch["smooth"]) + 1
    assert abs(c - (ev["res"] + ev["smooth"])) <= E.gamma(D + E.SLACK) * (ev["res_abs"] + ev["smooth_abs"]), name
    E.check_sums(None, None, g, ev, (ch["res"], ch["smooth"], ch["grad"]))
    # and the float gain itself: the same outputs as with the gain rounded by hand
    (r1, s1), g1 = _dev_pair(env, sd, images, mask, E.as_c_float(gain))
    assert c == r1 + s1 and np.array_equal(g, g1)


@pytest.mark.parametrize("name", list(E.FIELD_CASES))
def test_fused_pair_equals_separate_evaluations(env, name):
    sd, images, mask, gain, _ = E.field_case(name)
    pairs = ((1, 2), (0, 1)) if len(images) == 3 else ((0, 1),)
    res = smo = grad = None
    for a, b in pairs:
        r, s, g = _dev_cost(env, sd, images[a], images[b], mask, gain)
        res, smo, grad = (r, s, g) if res is None else (res + r, smo + s, grad + g)
    (r, s), g = _dev_pair(env, sd, images, mask, gain)
    assert _bits(r) == _bits(res) and _bits(s) == _bits(smo), name
    assert_bits_equal(g, grad, name)


def _warp_fields(nx, ny, rng):
    """pixel displacement fields (2, nx, ny): sources beyond every border, exact integers (landing on the
    last row and column and clamping past them), and sources exactly on the last row / column"""
    x = np.arange(nx, dtype=np.float64)[:, None] + np.zeros((1, ny))
    y = np.arange(ny, dtype=np.float64)[None, :] + np.zeros((nx, 1))
    yield "clamp", np.stack([rng.uniform(-1, 1, (nx, ny)) * nx, rng.uniform(-1, 1, (nx, ny)) * ny])
    yield "integer", np.stack([rng.integers(-3, 4, (nx, ny)), rng.integers(-3, 4, (nx, ny))]).astype(np.float64)
    yield "on last", np.stack([x - (nx - 1), y - (ny - 1)])
    yield "on last x, fractional y", np.stack([x - (nx - 1), rng.uniform(-0.99, 0.99, (nx, ny))])


@pytest.mark.parametrize("nx,ny", [(1, 1), (1, 7), (5, 1), (33, 40), (64, 31)])
def test_warp_bit_for_bit(env, nx, ny):
    torch, L, _ = env
    rng = np.random.default_rng(nx * 100 + ny)
    img = 10 * rng.random((nx, ny))
    for mask in (np.zeros((nx, ny), np.int8), (rng.random((nx, ny)) < 0.2).astype(np.int8)):
        for label, disp in _warp_fields(nx, ny, rng):
            d = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (img, mask, disp)]
            out = torch.empty((nx, ny), dtype=torch.float64, device="cuda")
            om = torch.empty((nx, ny), dtype=torch.int8, device="cuda")
            gr = torch.empty((2, nx, ny), dtype=torch.float64, device="cuda")
            L.call("b200_vet_warp", d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), nx, ny, out.data_ptr(),
                   om.data_ptr(), gr.data_ptr(), _stream(torch))
            o, m, g = ora.warp(img, mask, disp, gradient=True)
            what = f"{nx}x{ny} {label} mask={int(mask.any())}"
            assert_bits_equal(out.cpu().numpy(), o, what + " image")
            assert np.array_equal(om.cpu().numpy(), m), what + " mask"
            assert_bits_equal(gr.cpu().numpy(), g, what + " gradient")


@pytest.mark.parametrize("c,h,w,oh,ow", [(2, 3, 5, 1, 1), (2, 3, 5, 1, 9), (2, 3, 5, 9, 1), (1, 1, 1, 1, 4),
                                         (2, 32, 32, 1, 2048), (2, 32, 16, 504, 1)])
def test_zoom_at_one_row_or_column(env, c, h, w, oh, ow):
    """oh = 1 or ow = 1: the scale along that axis is 0 and every output samples the first row / column"""
    torch, L, _ = env
    a = np.random.default_rng(h * w + oh).normal(size=(c, h, w))
    out = torch.empty((c, oh, ow), dtype=torch.float64, device="cuda")
    L.call("b200_zoom_bilinear", torch.from_numpy(a).cuda().data_ptr(), c, h, w, oh, ow, out.data_ptr(),
           _stream(torch))
    assert_bits_equal(out.cpu().numpy(), ora.zoom_o1(a, oh, ow), f"zoom {(c, h, w, oh, ow)}")
