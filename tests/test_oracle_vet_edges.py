"""CPU tests: the NumPy restatement of tests/vet_edges.py against the C oracle (oracle/vet.py + vet_oracle.c) on
the VET edge grid --
  - single-pixel probes bit for bit: the residual and every gradient component (the pixel's term in the four
    sectors of its cell, zeros elsewhere), smoothness off; with a smoothness gain the residual bit for bit
    and the rest within the bound of its sums;
  - whole fields: each output of the oracle within gamma_D * sum |term| of the exact sum, D being the
    oracle's sequential chain (the number of terms);
and the grid's bookkeeping: it reaches every strip regime of vet_launch on an H100 SXM, every landing of the
warp and every mask, gain and frame count it is there for."""
import numpy as np
import pytest

import vet_edges as E
from oracle import vet as ora

SMS = E.H100_SXM_SMS


def test_grid_covers_every_strip_regime():
    reached = {}
    for geo, (nx, ny, xs, ys) in E.GEOMETRIES.items():
        for r in E.partition(nx, ny, xs, ys, SMS)["regimes"]:
            reached.setdefault(r, []).append(geo)
    assert set(reached) >= E.REGIMES, sorted(E.REGIMES - set(reached))
    # the bench's own levels: 2, 5, 118 and 512 strips on 132 SMs
    assert [E.partition(*E.GEOMETRIES[g], SMS)["strips"] for g in E.BENCH] == [2, 5, 118, 512]


def test_partition_covers_each_band_once():
    """strips tile each band's rows in order, trailing strips empty, and the bands tile the frame"""
    for geo, (nx, ny, xs, ys) in E.GEOMETRIES.items():
        for sms in (SMS, 114, 1):
            p = E.partition(nx, ny, xs, ys, sms)
            assert p["rows"][0][0] == 0 and p["rows"][-1][1] == nx
            assert all(a[1] == b[0] for a, b in zip(p["rows"], p["rows"][1:]))
            for l in range(p["ncx"]):
                sr = E.strip_rows(p, l)
                assert len(sr) == p["used"][l] <= p["strips"]
                assert sr[0][0] == p["rows"][l][0] and sr[-1][1] == p["rows"][l][1] - 1


@pytest.mark.parametrize("geo", list(E.GEOMETRIES))
def test_probe_grid_reaches_its_branches(geo):
    pts = E.probe_points(geo, SMS, geo not in E.BENCH)
    got = E.probe_branches(geo, pts, SMS)
    # every geometry: a skipped gradient row, clamps on every border, an integer landing
    assert {"skipped row", "x_low", "x_high", "y_low", "y_high"} <= got, sorted(got)
    assert {"x_integer", "y_integer"} & got
    nx, ny, xs, ys = E.GEOMETRIES[geo]
    p = E.partition(nx, ny, xs, ys, SMS)
    if any(u > 1 for u in p["used"]):
        assert "last strip first row" in got
    if any(u < p["strips"] for u in p["used"]):
        assert "band with empty trailing strips" in got


def test_probe_grid_reaches_every_landing():
    got = set()
    for geo in E.GEOMETRIES:
        got |= E.probe_branches(geo, E.probe_points(geo, SMS, geo not in E.BENCH), SMS)
    assert {"x_integer", "y_integer", "x_on_last", "y_on_last", "band with empty trailing strips"} <= got, sorted(got)


def _probes(geo):
    """every probe of the small geometries; three of each 2048^2 level (the oracle takes ~1 s there)"""
    pts = E.probe_points(geo, SMS, geo not in E.BENCH)
    return pts if geo not in E.BENCH else [pts[0], pts[len(pts) // 2], pts[-1]]


@pytest.mark.parametrize("geo", list(E.GEOMETRIES))
def test_probes_equal_oracle_bit_for_bit(geo):
    for pt in _probes(geo):
        sd, templ, inp, mask = E.probe_case(geo, pt)
        res, grad, _ = E.probe_expect(geo, pt, sd, templ, inp, mask)
        r, s = ora.cost_function(sd, templ, inp, mask, 0.0)
        g = ora.cost_function(sd, templ, inp, mask, 0.0, gradient=True)
        assert np.float64(r).view(np.int64) == np.float64(res).view(np.int64), (geo, pt, r, res)
        assert s == 0.0
        assert np.array_equal(g, grad), (geo, pt, np.argwhere(g != grad)[:4].tolist())
        if geo in E.BENCH:
            continue
        # with the smoothness term: the residual unchanged, the gradient within the bound of its sums
        ev = E.probe_eval(geo, pt, sd, templ, inp, mask, 1e6)
        r, s = ora.cost_function(sd, templ, inp, mask, 1e6)
        g = ora.cost_function(sd, templ, inp, mask, 1e6, gradient=True)
        assert np.float64(r).view(np.int64) == np.float64(res).view(np.int64)
        E.check_sums(r, s, g, ev, E.oracle_chains(ev))


_REACH = {"sub": {"|d| < 1"}, "clamp": {"clamp x both sides", "clamp y both sides"},
          "integer": {"integer displacements", "lands on last x", "lands on last y"}}


def test_field_grid_covers_masks_gains_frames():
    kinds = {k: {c[i] for c in E.FIELD_CASES.values()} for k, i in (("disp", 1), ("mask", 2), ("gain", 3),
                                                                     ("T", 4))}
    assert kinds == dict(disp=set(_REACH), mask={"clear", "all", "patch"}, gain=set(E.GAINS), T={2, 3})
    assert {c[0] for c in E.FIELD_CASES.values()} == set(E.GEOMETRIES)


@pytest.mark.parametrize("name", list(E.FIELD_CASES))
def test_fields_oracle_within_bound_of_exact(name):
    sd, images, mask, gain, geo = E.field_case(name)
    pairs = ((1, 2), (0, 1)) if len(images) == 3 else ((0, 1),)
    for a, b in pairs:
        ev = E.evaluate(sd, images[a], images[b], mask, gain)
        kind, mkind = E.FIELD_CASES[name][1], E.FIELD_CASES[name][2]
        got = E.field_branches(name, ev["px"])
        assert _REACH[kind] <= got, (name, sorted(got))
        if mkind == "patch" and kind != "integer":
            assert "fractional mask" in got
        if mkind == "all":
            assert ev["res_abs"] == 0.0 and not ev["grad"].any()
        r, s = ora.cost_function(sd, images[a], images[b], mask, gain)
        g = ora.cost_function(sd, images[a], images[b], mask, gain, gradient=True)
        E.check_sums(r, s, g, ev, E.oracle_chains(ev))
