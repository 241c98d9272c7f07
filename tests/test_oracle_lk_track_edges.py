"""CPU tests: the tracker oracle (oracle/lucaskanade.py + lk_oracle.c) against live cv2 on the edge grid of
tests/lk_track_edges.py -- EVERY point's next position bit for bit (NaN where cv2 has NaN) and its status,
lost points included -- and the pyramid and Scharr levels against cv2.buildOpticalFlowPyramid.  The GPU
machines have no cv2; these pins are what make the oracle the arbiter of tests/test_lk_track_edges_gpu.py."""
import numpy as np
import pytest
from conftest import assert_bits_equal

import lk_track_edges as edges
from oracle import lucaskanade as ora

cv2 = pytest.importorskip("cv2")


def _cv2_track(I, J, pts, win, levels, criteria, min_eig):
    p1, st, _ = cv2.calcOpticalFlowPyrLK(I, J, pts, None, winSize=win, maxLevel=levels, criteria=criteria,
                                         flags=0, minEigThreshold=min_eig)
    return p1.reshape(-1, 2), st.ravel()


@pytest.mark.parametrize("tag", list(edges.CASES))
def test_oracle_tracker_equals_cv2_on_every_point(tag):
    I, J, pts, c = edges.case_inputs(tag)
    want, wst = _cv2_track(I, J, pts, c["win"], c["levels"], c["criteria"], c["min_eig"])
    got, gst = ora.calc_optical_flow_pyr_lk(I, J, pts, c["win"], c["levels"], c["criteria"], c["min_eig"])
    assert np.array_equal(gst, wst), f"status: {int((gst != wst).sum())} of {len(wst)} differ"
    assert_bits_equal(got, want, "next points")
    # the special points are lost on both sides, with their coordinates carried through the levels
    assert not wst[-len(edges.SPECIAL):-3].any()


def test_grid_reaches_its_branches():
    """The grid is only worth its name if the cases take the branches they are named for."""
    def st(tag):
        I, J, pts, c = edges.case_inputs(tag)
        return _cv2_track(I, J, pts, c["win"], c["levels"], c["criteria"], c["min_eig"])
    # a ninth level changes which points cv2 tracks at 1024^2, 3x3
    p7, s7 = st("tex1024-w3x3-L7-c3_10_0-e0.0001")
    p8, s8 = st("tex1024-w3x3-L8-c3_10_0-e0.0001")
    p10, s10 = st("tex1024-w3x3-L10-c3_10_0-e0.0001")
    assert not np.array_equal(s7, s8) and np.array_equal(s8, s10)
    assert_bits_equal(p8, p10, "nr_levels 8 and 10 build the same nine levels")
    # max_count 0 leaves every point where the coarsest level put it; more iterations change points
    p0, s0 = st("tex300x340-w21x21-L3-c3_0_0-e0.0001")
    p1, _ = st("tex300x340-w21x21-L3-c3_1_0-e0.0001")
    p100, _ = st("tex300x340-w21x21-L3-c3_100_0-e0.0001")
    p500, _ = st("tex300x340-w21x21-L3-c3_500_0-e0.0001")
    assert not np.array_equal(p0, p1) and not np.array_equal(p1, p100)
    assert_bits_equal(p100, p500, "max_count is clamped to 100")
    # the flat frame loses every point through D / minEig, the saturated shift tracks none either
    assert not st("flat64x80-w21x21-L2-c3_10_0-e0.0001")[1].any()
    # min_eig_thr 1e-2 loses points that 1e-3 keeps
    assert st("tex300x340-w21x21-L3-c3_10_0-e0.01")[1].sum() < st("tex300x340-w21x21-L3-c3_10_0-e0.001")[1].sum()
    # the -0.0 points are tracked like any other point
    assert st("tex300x340-w64x64-L2-c3_10_0-e0.0001")[1][-3:].all()


@pytest.mark.parametrize("win", [(65, 65), (30, 100), (2, 2), (2, 9), (9, 2), (3, 3)])
def test_oracle_beyond_the_device_windows_and_cv2_refusals(win):
    """Windows above 4096 pixels: cv2 tracks them and so does the oracle (the device refuses them with
    NotImplementedError).  Sides below 3 and negative level counts: cv2 raises its assertion, whose text
    the product's ValueError repeats."""
    from pysteps_b200.motion.lucaskanade import _tracker_args
    I, J = edges.frames("tex300x340")
    pts = ora.good_features_to_track(I, None, 60, 0.01, 7)
    for levels in (2, -1):
        if win[0] > 2 and win[1] > 2 and levels >= 0:
            want, wst = _cv2_track(I, J, pts, win, levels, (3, 10, 0), 1e-4)
            got, gst = ora.calc_optical_flow_pyr_lk(I, J, pts, win, levels, (3, 10, 0), 1e-4)
            assert np.array_equal(gst, wst) and wst.sum() > 30
            assert_bits_equal(got, want, f"{win}")
            continue
        with pytest.raises(cv2.error) as cv_err:
            _cv2_track(I, J, pts, win, levels, (3, 10, 0), 1e-4)
        with pytest.raises(ValueError) as our_err:
            _tracker_args(win, levels, (3, 10, 0))
        assert str(our_err.value) in str(cv_err.value)


@pytest.mark.parametrize("shape,win,levels", [
    ((37, 53), (5, 5), 4), ((300, 340), (21, 21), 3), ((1, 1), (3, 3), 2), ((7, 5), (3, 3), 3),
    ((11, 11), (3, 3), 5), ((24, 26), (5, 5), 6),   # level 2 is 6x7: one pixel above the window
    ((20, 22), (5, 5), 6),                          # level 2 would be 5x6: stops at the window
    ((41, 7), (3, 3), 6), ((1024, 1024), (3, 3), 10), ((513, 1025), (3, 3), 12)])
def test_pyramid_and_scharr_levels_equal_cv2(shape, win, levels):
    rng = np.random.default_rng(shape[0] * 7919 + shape[1])
    a = rng.integers(0, 256, shape).astype(np.uint8)
    n, pyr = cv2.buildOpticalFlowPyramid(a, win, levels, withDerivatives=True)
    sizes = edges.pyramid_sizes(shape[0], shape[1], win, levels)
    assert n == len(sizes) - 1, "level count"
    lev = a
    for lvl in range(n + 1):
        assert pyr[2 * lvl].shape == sizes[lvl]
        assert np.array_equal(pyr[2 * lvl], lev), f"level {lvl}"
        assert np.array_equal(pyr[2 * lvl + 1], ora.scharr_deriv(lev)), f"Scharr level {lvl}"
        lev = ora.pyr_down(lev)
