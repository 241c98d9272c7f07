"""GPU tests of the pyramidal LK tracker (csrc/lk_track.cu) on the edge grid of tests/lk_track_edges.py:
windows with no 8-pixel chunk or no scalar tail, the largest shared-memory footprints and divisors beyond 64,
level counts from 0 to more than the eight the level arrays once held, every criteria branch and clamp,
frames smaller than the window, flat and saturated frames, window origins on the bounds, NaN / inf / huge
coordinates.  Bars, against the oracle (pinned to cv2 on the same grid by tests/test_oracle_lk_track_edges.py):
every Gaussian and Scharr level bit-identical, every point's next position bit-identical (NaN where the oracle
has NaN; NaN payloads are not compared) and every status equal, lost points included."""
import numpy as np
import pytest
from conftest import assert_bits_equal

import lk_track_edges as edges

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a GPU"
    from pysteps_b200 import _device, _lib
    _device.require_cuda()
    return torch, _lib


def _pyramid(env, img, win, levels, deriv):
    """b200_lk_build_pyramid of a uint8 image -> (levels tensor, Scharr tensor or None, coarsest level)"""
    torch, L = env
    from pysteps_b200.motion.lucaskanade import _pyramid_layout
    m, n = img.shape
    lv, total = _pyramid_layout(m, n, win, levels)
    P = torch.empty(total, dtype=torch.uint8, device="cuda")
    D = torch.empty(2 * total, dtype=torch.int16, device="cuda") if deriv else None
    src = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    L.call("b200_lk_build_pyramid", src.data_ptr(), m, n, win[0], win[1], levels, P.data_ptr(),
           None if D is None else D.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return P, D, lv


def _check_levels(P, D, lv, img, win, levels, what):
    from oracle import lucaskanade as ora
    sizes = edges.pyramid_sizes(img.shape[0], img.shape[1], win, levels)
    assert lv == len(sizes) - 1, f"{what}: coarsest level {lv}, cv2 builds {len(sizes) - 1}"
    P = P.cpu().numpy()
    D = None if D is None else D.cpu().numpy()
    lev, off = img, 0
    for lvl, (h, w) in enumerate(sizes):
        assert np.array_equal(P[off:off + h * w].reshape(h, w), lev), f"{what}: level {lvl} ({h}x{w})"
        if D is not None:
            assert np.array_equal(D[2 * off:2 * (off + h * w)].reshape(h, w, 2), ora.scharr_deriv(lev)), \
                f"{what}: Scharr level {lvl} ({h}x{w})"
        off += h * w
        lev = ora.pyr_down(lev)
    assert off == P.size


def _track(env, pyrs, shape, pts, c, count=None):
    """b200_lk_track with the criteria clamped as the product clamps them; count: the device count
    (npts_dev) instead of all points.  Outputs start as a sentinel so untouched entries show."""
    torch, L = env
    from pysteps_b200.motion.lucaskanade import _tracker_args
    (PI, DI, _), (PJ, _, _) = pyrs
    win_w, win_h, levels, max_count, eps = _tracker_args(c["win"], c["levels"], c["criteria"])
    npts = len(pts)
    p0 = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    p1 = torch.full((npts, 2), -1234.5, dtype=torch.float32, device="cuda")
    st = torch.full((npts,), 7, dtype=torch.uint8, device="cuda")
    cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
    L.call("b200_lk_track", PI.data_ptr(), PJ.data_ptr(), DI.data_ptr(), shape[0], shape[1], win_w, win_h,
           levels, max_count, eps, float(c["min_eig"]), p0.data_ptr(), npts,
           None if cnt is None else cnt.data_ptr(), p1.data_ptr(), st.data_ptr(),
           torch.cuda.current_stream().cuda_stream)
    return p1.cpu().numpy(), st.cpu().numpy()


def _run(env, tag, count=None):
    from oracle import lucaskanade as ora
    I, J, pts, c = edges.case_inputs(tag)
    pyrs = (_pyramid(env, I, c["win"], c["levels"], True), _pyramid(env, J, c["win"], c["levels"], False))
    got, gst = _track(env, pyrs, I.shape, pts, c, count)
    want, wst = ora.calc_optical_flow_pyr_lk(I, J, pts, c["win"], c["levels"], c["criteria"], c["min_eig"])
    return I, J, pts, c, pyrs, (got, gst), (want, wst)


@pytest.mark.parametrize("tag", list(edges.CASES))
def test_tracker_equals_oracle_on_every_point(env, tag):
    I, J, pts, c, pyrs, (got, gst), (want, wst) = _run(env, tag)
    _check_levels(*pyrs[0], I, c["win"], c["levels"], "I")
    _check_levels(*pyrs[1], J, c["win"], c["levels"], "J")
    bad = np.nonzero(gst != wst)[0]
    assert bad.size == 0, f"status of {bad.size} of {len(pts)} points differs, e.g. {pts[bad[:4]].tolist()}"
    assert_bits_equal(got, want, f"next points of {tag}")


def test_device_count_below_npts(env):
    """npts_dev: only the first *npts_dev points are tracked (a count above npts is npts); the rest of
    next_pts and status is not written."""
    tag = "tex300x340-w16x16-L2-c3_10_0-e0.0001"
    I, J, pts, c, pyrs, _, (want, wst) = _run(env, tag)
    for count in (len(pts) - 37, 1, 0, len(pts) + 5):
        got, gst = _track(env, pyrs, I.shape, pts, c, count)
        k = min(count, len(pts))
        assert np.array_equal(gst[:k], wst[:k]), count
        assert_bits_equal(got[:k], want[:k], f"count {count}")
        assert (gst[k:] == 7).all() and (got[k:] == -1234.5).all(), f"count {count}: points past it written"


def test_dense_lucaskanade_tracks_nine_levels(env):
    """dense_lucaskanade at 1024^2 with a 3x3 window and nr_levels=10 builds and tracks the nine levels cv2
    builds (at seven levels the sparse vectors differ): sparse vectors bit-identical, dense field <= 1e-12."""
    from oracle import lucaskanade as ora
    from pysteps_b200 import _synthetic as syn
    from pysteps_b200.motion.lucaskanade import dense_lucaskanade as lk
    fr = syn.rain_frames(1024, 1024, 2, 5)
    kw = dict(lk_kwargs={"winsize": (3, 3), "nr_levels": 10})
    xy, uv = lk(fr, dense=False, **kw)
    oxy, ouv = ora.dense_lucaskanade(fr, dense=False, **kw)
    assert np.array_equal(xy, oxy) and np.array_equal(uv, ouv)
    sxy, suv = ora.dense_lucaskanade(fr, dense=False, lk_kwargs={"winsize": (3, 3), "nr_levels": 7})
    assert not (np.array_equal(sxy, oxy) and np.array_equal(suv, ouv)), "the case must depend on levels 8+"
    V = lk(fr, **kw)
    Vo = ora.dense_lucaskanade(fr, **kw)
    assert V.shape == Vo.shape and np.abs(V - Vo).max() <= 1e-12
