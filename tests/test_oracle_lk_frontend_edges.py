"""CPU tests: the front-end and eigenvalue-map oracles (oracle/lucaskanade.py + lk_oracle.c) pinned on the
edge grid of tests/lk_frontend_edges.py --
  - ora.corner_min_eigen_val against cv2.cornerMinEigenVal(q, 5, ksize=3), bit for bit;
  - ora.morph_open_cross3 and ora.dilate_rect against cv2.morphologyEx / cv2.dilate;
  - ora.morph_opening, ora.detection_image and ora.tracking_image against the reference itself: the uint8
    image and mask pysteps hands to cv2.goodFeaturesToTrack / cv2.calcOpticalFlowPyrLK, captured by
    patching those two names;
and the grid's own bookkeeping: every case reaches the branches it names, and the grid reaches every
branch, each case being the only one there for at least one of them.  The GPU machines have no cv2;
these pins are what make the oracle the arbiter of tests/test_lk_frontend_edges_gpu.py."""
import numpy as np
import pytest
from conftest import assert_bits_equal

import lk_frontend_edges as edges
from oracle import lucaskanade as ora


def _cv2():
    return pytest.importorskip("cv2")


def _avx512():
    try:
        with open("/proc/cpuinfo") as f:
            return " avx512f" in f.read()
    except OSError:
        return False


@pytest.mark.parametrize("cases,required,branches", [
    (edges.FRONT_CASES, edges.FRONT_REQUIRED, edges.front_branches),
    (edges.EIG_CASES, edges.EIG_REQUIRED, edges.eig_branches)], ids=["front", "eig"])
def test_grid_covers_every_branch(cases, required, branches):
    """Each case reaches what it names; the names cover every required branch; every case is the only one
    to name at least one of them, so removing a case uncovers a branch."""
    named = set()
    for tag, c in cases.items():
        reached = branches(tag)
        assert c["why"] <= reached, f"{tag} does not reach {sorted(c['why'] - reached)}"
        assert c["why"] <= required, f"{tag} names branches outside the required set: {sorted(c['why'] - required)}"
        others = set().union(*(d["why"] for t, d in cases.items() if t != tag))
        assert c["why"] - others, f"{tag} is not the only case for any of its branches"
        named |= c["why"]
    assert named >= required, f"uncovered: {sorted(required - named)}"


def test_classifier_tiles_per_cta():
    """nparts = min(tiles, 4 x SMs) persistent CTAs: the tile-count cases give 1, 1, 2, 3 and 5 tiles per
    CTA, and the ring's parity is 0, 0, 1, 1, 0 over a CTA's tiles"""
    for sms in (edges.H100_SXM_SMS, 114, 1):
        per = {}
        for kind in ("tall", "wide"):
            for step, want in (("nparts-1", 1), ("nparts", 1), ("nparts+1", 2), ("2nparts+1", 3), ("4nparts+1", 5)):
                m, n = edges.front_shape(f"{kind}-{step}", sms)
                t = edges._tiles(m, n)
                assert t == 4 * sms + edges._TILE_STEPS[step](4 * sms)
                per[kind, step] = -(-t // min(t, 4 * sms))
                assert per[kind, step] == want, (sms, kind, step)
    assert [(it >> 1) & 1 for it in range(5)] == [0, 0, 1, 1, 0]


def test_chain_rounds():
    """box_chain's interior rounds start at h = BOX_R + BOX_U + 2 = 74"""
    assert edges.chain_rounds(73) == (0, 73)
    assert edges.chain_rounds(74) == (1, 66)
    assert edges.chain_rounds(81) == (1, 73) and edges.chain_rounds(82) == (2, 66)
    assert edges.chain_rounds(4099) == (504, 67)


@pytest.mark.parametrize("tag", list(edges.EIG_CASES))
def test_min_eig_oracle_equals_cv2(tag):
    cv2 = _cv2()
    if not _avx512():
        pytest.skip("the oracle restates cv2's AVX-512 build; this host has no avx512f")
    q = edges.eig_input(tag)
    assert_bits_equal(ora.corner_min_eigen_val(q), cv2.cornerMinEigenVal(q, 5, ksize=3), tag)


def _binary(tag):
    a, um, _, _ = edges.front_inputs(tag)
    ma = edges.masked_frame(np.asarray(a, np.float64), um)
    return (ma.filled(ma.min()) > ma.min()).astype(np.uint8), np.ma.getmaskarray(ma).astype(np.uint8)


@pytest.mark.parametrize("tag", list(edges.FRONT_CASES))
def test_opening_and_dilation_oracles_equal_cv2(tag):
    cv2 = _cv2()
    b, mask = _binary(tag)
    kernel = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (3, 3))
    assert np.array_equal(ora.morph_open_cross3(b), cv2.morphologyEx(b, cv2.MORPH_OPEN, kernel)), "opening"
    k = edges.FRONT_CASES[tag]["buffer_mask"]
    for kk in {k, 1, 2, 5} - {0}:
        assert np.array_equal(ora.dilate_rect(mask, kk), cv2.dilate(mask, np.ones((kk, kk), np.uint8), 1)), kk


@pytest.fixture(scope="module")
def reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _cv2()
    return (_refimport.ref_module("pysteps.utils.images"), _refimport.ref_module("pysteps.feature.shitomasi"),
            _refimport.ref_module("pysteps.tracking.lucaskanade"))


def _capture(monkeypatch, module, name):
    """patch cv2.<name> as the reference module sees it: record the image and mask, return no points"""
    got = {}

    def fake(*args, **kwargs):
        got["image"] = np.array(args[0], copy=True)
        got["mask"] = kwargs.get("mask")
        if name == "calcOpticalFlowPyrLK":
            p0 = args[2]
            return p0.copy(), np.zeros((len(p0), 1), np.uint8), np.zeros((len(p0), 1), np.float32)
        return None

    monkeypatch.setattr(module.cv2, name, fake)
    return got


@pytest.mark.parametrize("tag", list(edges.FRONT_CASES))
def test_front_oracles_equal_reference(tag, reference, monkeypatch):
    images, shitomasi, tracking = reference
    a, um, _, c = edges.front_inputs(tag)
    ma = edges.masked_frame(a, um)
    if c["opening"]:
        want = images.morph_opening(ma.copy(), ma.min(), 3)
        got = ora.morph_opening(ma.copy(), ma.min(), 3)
        assert np.array_equal(np.ma.getmaskarray(got), np.ma.getmaskarray(want))
        assert_bits_equal(np.ma.getdata(got), np.ma.getdata(want), "opened image")
        ma = got
    det = _capture(monkeypatch, shitomasi, "goodFeaturesToTrack")
    shitomasi.detection(ma, buffer_mask=c["buffer_mask"])
    q, valid = ora.detection_image(ma, c["buffer_mask"])
    assert np.array_equal(q, det["image"]), "detection image"
    assert np.array_equal(valid, det["mask"]), "validity mask"
    trk = _capture(monkeypatch, tracking, "calcOpticalFlowPyrLK")
    tracking.track_features(ma, ma, np.array([[0.0, 0.0]], np.float32))
    assert np.array_equal(ora.tracking_image(ma), trk["image"]), "tracking image"
