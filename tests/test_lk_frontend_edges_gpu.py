"""GPU tests of the dense LK front end and the Shi-Tomasi eigenvalue map on the edge grid of
tests/lk_frontend_edges.py, every comparison bit for bit:
  - the stage kernels of csrc/lk_dense.cu against the oracle: mask, opened image, the 12 statistics,
    the tracker's and the detector's uint8 images and the validity map;
  - the fused front end (csrc/lk_frontend.cu) against the stage kernels on the same outputs, given the
    case's user mask (an all-clear one where the case has none) and given no user-mask pointer;
  - b200_min_eig against the oracle's cv::cornerMinEigenVal (pinned to cv2 on the same grid by
    tests/test_oracle_lk_frontend_edges.py);
  - dense_lucaskanade against the oracle at a few grid shapes, and on a frame stack that starts 8 bytes
    past a 16-byte boundary.
The tile-count cases are sized from the SM count of the device at hand."""
import numpy as np
import pytest
from conftest import assert_bits_equal

import lk_frontend_edges as edges
from oracle import lucaskanade as ora

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _lib, torch.cuda.get_device_properties(0).multi_processor_count


def _upload(torch, a, offset=0):
    """a float64 CUDA copy of `a` starting `offset` elements into its allocation"""
    flat = np.ascontiguousarray(a, np.float64).ravel()
    base = torch.empty(flat.size + offset, dtype=torch.float64, device="cuda")
    t = base[offset:]
    t.copy_(torch.from_numpy(flat))
    return t


def _stages(env, img, um, m, n, opening, buffer_mask, flag):
    torch, L, _ = env
    s = torch.cuda.current_stream().cuda_stream
    u8 = lambda: torch.full((m, n), 77, dtype=torch.uint8, device="cuda")  # noqa: E731
    mask, q_track, q_det, valid = u8(), u8(), u8(), u8()
    st0 = torch.full((3,), -1.0, dtype=torch.float64, device="cuda")
    st = torch.full((12,), -1.0, dtype=torch.float64, device="cuda")
    L.call("b200_mask_invalid", img.data_ptr(), None if um is None else um.data_ptr(), m, n, mask.data_ptr(),
           st0.data_ptr(), s)
    opened = img
    if opening:
        opened = torch.full((m * n,), -1.0, dtype=torch.float64, device="cuda")
        L.call("b200_morph_opening", img.data_ptr(), mask.data_ptr(), m, n, 3, st0.data_ptr(), st0.data_ptr(),
               opened.data_ptr(), s)
    L.call("b200_masked_minmax", opened.data_ptr(), mask.data_ptr(), m, n, buffer_mask, st0.data_ptr(),
           st.data_ptr(), s)
    L.call("b200_quantise_u8", opened.data_ptr(), mask.data_ptr(), m, n, 0 | flag, 0, st.data_ptr(), st.data_ptr(),
           q_track.data_ptr(), None, s)
    L.call("b200_quantise_u8", opened.data_ptr(), mask.data_ptr(), m, n, 1 | flag, buffer_mask, st.data_ptr(),
           st.data_ptr(), q_det.data_ptr(), valid.data_ptr(), s)
    out = dict(mask=mask, st0=st0, st=st, q_track=q_track, q_det=q_det, valid=valid)
    out = {k: v.cpu().numpy() for k, v in out.items()}
    out["opened"] = opened.cpu().numpy().reshape(m, n)
    return out


def _fused(env, img, um, m, n, opening, buffer_mask, flag):
    torch, L, _ = env
    s = torch.cuda.current_stream().cuda_stream
    u8 = lambda: torch.full((m, n), 77, dtype=torch.uint8, device="cuda")  # noqa: E731
    mask, q_track, q_det, valid = u8(), u8(), u8(), u8()
    st0 = torch.full((3,), -1.0, dtype=torch.float64, device="cuda")
    st = torch.full((12,), -1.0, dtype=torch.float64, device="cuda")
    L.call("b200_lk_frontend", img.data_ptr(), None if um is None else um.data_ptr(), m, n, opening, buffer_mask,
           flag, mask.data_ptr(), st0.data_ptr(), st.data_ptr(), q_track.data_ptr(), q_det.data_ptr(),
           valid.data_ptr(), s)
    out = dict(mask=mask, st0=st0, st=st, q_track=q_track, q_det=q_det, valid=valid)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(a, um, opening, buffer_mask):
    """what the reference computes from the frame: mask, opened image, statistics, both uint8 images"""
    ma = edges.masked_frame(a, um)
    mask = np.ma.getmaskarray(ma)
    opened = ora.morph_opening(ma, ma.min(), 3) if opening else ma
    data = np.ma.getdata(opened).astype(np.float64)
    vals = np.asarray(a, np.float64)[~mask]
    st0 = np.array([vals.min(), vals.max(), float(vals.size)])
    q_det, valid = ora.detection_image(opened, buffer_mask)
    return dict(mask=mask.astype(np.uint8), st0=st0, opened=data, st=edges.front_stats(data, mask, buffer_mask),
                q_track=ora.tracking_image(opened), q_det=q_det, valid=valid.astype(np.uint8))


def _compare(got, want, what, keys):
    for k in keys:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        if g.dtype.kind == "f":
            assert_bits_equal(g.reshape(w.shape), w, f"{what}: {k}")
        else:
            g = g.reshape(w.shape)
            bad = np.argwhere(g != w)
            assert bad.size == 0, f"{what}: {k}: {len(bad)} pixels differ, first at {bad[:4].tolist()}"


_ALL = ("mask", "st0", "st", "q_track", "q_det", "valid")


@pytest.mark.parametrize("tag", list(edges.FRONT_CASES))
def test_front_end_equals_oracle_and_stage_kernels(env, tag):
    torch, L, sms = env
    a, um, _, c = edges.front_inputs(tag, sms)
    m, n = a.shape
    op, b, flag = c["opening"], c["buffer_mask"], 2 if c["f32"] else 0
    br = edges.front_branches(tag, sms)
    assert c["why"] <= br, f"{tag} does not reach {sorted(c['why'] - br)} on {sms} SMs"
    img = _upload(torch, a, c["offset"])
    um_d = None if um is None else torch.from_numpy(um.astype(np.uint8)).cuda()
    zeros = torch.zeros((m, n), dtype=torch.uint8, device="cuda")
    want = _oracle(a, um, op, b)
    # with the case's user mask (all clear where it has none) and without a user-mask pointer
    for label, ptr in (("user mask", um_d if um_d is not None else zeros), ("no mask pointer", None)):
        got = _stages(env, img, ptr, m, n, op, b, flag)
        if ptr is um_d or um is None:
            _compare(got, want, f"{tag} stages ({label}) vs oracle", _ALL + ("opened",))
        if "path=fused" in br:
            _compare(_fused(env, img, ptr, m, n, op, b, flag), got, f"{tag} fused ({label}) vs stages", _ALL)


@pytest.mark.parametrize("tag", list(edges.EIG_CASES))
def test_min_eig_equals_oracle(env, tag):
    torch, L, _ = env
    c = edges.EIG_CASES[tag]
    assert c["why"] <= edges.eig_branches(tag)
    q = edges.eig_input(tag)
    h, w = q.shape
    qd = torch.from_numpy(q).cuda()
    eig = torch.full((h, w), -7.0, dtype=torch.float32, device="cuda")
    L.call("b200_min_eig", qd.data_ptr(), h, w, eig.data_ptr(), torch.cuda.current_stream().cuda_stream)
    got, want = eig.cpu().numpy(), ora.corner_min_eigen_val(q)
    if not np.array_equal(got.view(np.int32), want.view(np.int32)):
        bad = np.argwhere(got.view(np.int32) != want.view(np.int32))
        rows = sorted({int(y) for y, _ in bad})
        cols = sorted({int(x) for _, x in bad})
        raise AssertionError(f"{tag}: {len(bad)} pixels differ, rows {rows[:8]}..{rows[-1]}, "
                             f"columns {cols[:8]}..{cols[-1]}")


def test_grid_reaches_its_branches_on_this_device(env):
    """the grid covers every branch with the tile-count cases sized for the device at hand: one, two,
    three and five tiles per CTA"""
    _, _, sms = env
    reached = set().union(*(edges.front_branches(t, sms) for t in edges.FRONT_CASES))
    assert edges.FRONT_REQUIRED <= reached, sorted(edges.FRONT_REQUIRED - reached)
    print(f"{sms} SMs: nparts {4 * sms}, up to 5 tiles per CTA")


@pytest.mark.parametrize("m,n,T", [(16, 130, 2), (75, 129, 2), (138, 68, 3), (200, 202, 2), (33, 128, 2)])
def test_dense_lucaskanade_equals_oracle_at_grid_shapes(env, m, n, T):
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    fr = syn.rain_frames(m, n, T, m + n)
    kw = dict(fd_kwargs={"buffer_mask": 3}) if n % 2 else {}
    xy, uv = lk(fr, dense=False, **kw)
    oxy, ouv = ora.dense_lucaskanade(fr, dense=False, **kw)
    assert np.array_equal(xy, oxy) and np.array_equal(uv, ouv)
    V, Vo = lk(fr, **kw), ora.dense_lucaskanade(fr, **kw)
    assert V.shape == Vo.shape and np.abs(V - Vo).max() <= 1e-12


def test_dense_lucaskanade_on_a_view_8_bytes_off_alignment(env):
    """A contiguous float64 CUDA view whose first element sits 8 bytes past a 16-byte boundary (even
    width): the fused front end cannot stage it by TMA, so the stage kernels take it -- same sparse
    vectors and dense field as the oracle."""
    torch, _, _ = env
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    m, n = 120, 160
    fr = syn.rain_frames(m, n, 2, 17)
    base = torch.zeros(1 + 2 * m * n, dtype=torch.float64, device="cuda")
    view = base[1:1 + 2 * m * n].view(2, m, n)
    view.copy_(torch.from_numpy(fr))
    assert view.data_ptr() % 16 == 8 and view.is_contiguous()
    xy, uv = lk(view, dense=False)
    oxy, ouv = ora.dense_lucaskanade(fr, dense=False)
    assert len(oxy) > 0
    assert np.array_equal(xy.cpu().numpy(), oxy) and np.array_equal(uv.cpu().numpy(), ouv)
    V = lk(view).cpu().numpy()
    Vo = ora.dense_lucaskanade(fr)
    assert V.shape == Vo.shape and np.abs(V - Vo).max() <= 1e-12
