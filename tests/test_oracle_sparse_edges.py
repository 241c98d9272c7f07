"""CPU tests of the sparse-cleansing edge grid (tests/sparse_edges.py): every case takes the branches it
names, the oracle's detect_outliers and decluster equal the live reference on the whole grid (non-finite
and huge cells included), the vectorised decluster equals the oracle where the oracle's O(n * cells)
loop is affordable, no outlier decision of the grid is a tie at the threshold for want of a case, and
the device queries' pending-node heaps stay well inside their spill arena."""
import ctypes
import warnings

import numpy as np
import pytest

import sparse_edges as E
from oracle import lucaskanade as ora


def _reference():
    try:
        from _refimport import available, ref_module
    except ImportError:
        from golden._refimport import available, ref_module
    if not available():
        pytest.skip("the reference is not importable here")
    return ref_module("pysteps.utils.cleansing")


def _quiet():
    w = warnings.catch_warnings()
    w.__enter__()
    warnings.simplefilter("ignore")
    return w


def test_every_branch_is_named_and_taken():
    named = set()
    for tag, c in E.ALL_CASES.items():
        got = E.classify(tag)
        assert c["claims"], f"{tag} names no branch"
        missing = set(c["claims"]) - got
        assert not missing, f"{tag} names {sorted(missing)} but takes {sorted(got)}"
        named |= set(c["claims"])
    for op, branches in E.BRANCHES.items():
        unnamed = set(branches) - named
        assert not unnamed, f"{op}: no case names {sorted(unnamed)}"
    assert named <= {b for bs in E.BRANCHES.values() for b in bs}, named


@pytest.mark.parametrize("tag", list(E.GLOBAL))
def test_global_outlier_oracle_equals_reference(tag):
    cl = _reference()
    uv = E.global_inputs(tag)
    c = E.GLOBAL[tag]
    w = _quiet()
    try:
        want = cl.detect_outliers(uv.copy(), c["thr"])
        got = ora.detect_outliers(uv.copy(), c["thr"])
    finally:
        w.__exit__(None, None, None)
    assert np.array_equal(got, want)
    md, sing, cond = E.md_extended(uv) if len(uv) >= 2 else (np.zeros(0), np.zeros(0, bool), np.zeros(0))
    if E.global_lu(uv) in ("p0=0", "u22=0", "collinear"):
        assert sing.all() and not want.any()  # LinAlgError: MD = 0 everywhere
    elif len(uv) >= 2:
        # the extended-precision distance decides every row outside the margin
        tie = E.tie_rows(md, sing, cond, c["thr"])
        assert tie.sum() < max(len(uv), 1)
        assert np.array_equal(want[~tie], (md > c["thr"])[~tie])
        assert 0 < want.sum() < len(uv), "a grid case with nothing (or everything) to flag"


@pytest.mark.parametrize("tag", list(E.KNN))
def test_knn_outlier_oracle_equals_reference(tag):
    cl = _reference()
    xy, uv = E.knn_inputs(tag)
    c = E.KNN[tag]
    w = _quiet()
    try:
        want = cl.detect_outliers(uv.copy(), c["thr"], xy.copy(), c["k"])
        with ora.knn_mode("ckdtree"):
            got = ora.detect_outliers(uv.copy(), c["thr"], xy.copy(), c["k"])
    finally:
        w.__exit__(None, None, None)
    assert np.array_equal(got, want)
    if len(xy) < 2:
        return
    inds = E.knn_neighbours(xy, c["k"])
    md, sing, cond = E.md_extended(uv, inds)
    tie = E.tie_rows(md, sing, cond, c["thr"])
    assert tie.sum() < len(xy), f"{int(tie.sum())} tie rows of {len(xy)}"
    assert np.array_equal(want[~tie], (md > c["thr"])[~tie]), np.nonzero(want[~tie] != (md > c["thr"])[~tie])
    if "k:sing_identical" in c["claims"] or "k:sing_constv" in c["claims"]:
        assert sing.sum() >= 50 and not want[sing].any()


@pytest.mark.parametrize("tag", list(E.DECLUSTER))
def test_decluster_oracle_equals_reference(tag):
    cl = _reference()
    c = E.DECLUSTER[tag]
    xy, uv = E.decluster_inputs(c)
    w = _quiet()
    try:
        with np.errstate(all="ignore"):
            want = cl.decluster(xy.copy(), uv.copy(), c["scale"], c["min_samples"])
        if c["n"] <= 4096:  # the oracle's loop over cells
            with np.errstate(all="ignore"):
                got = ora.decluster(xy.copy(), uv.copy(), c["scale"], c["min_samples"])
            assert np.array_equal(got[0], want[0], equal_nan=True) and np.array_equal(got[1], want[1], equal_nan=True)
    finally:
        w.__exit__(None, None, None)
    if E.decluster_refused(xy, c["scale"], c["min_samples"]):
        return
    vec = E.decluster_vectorised(xy, uv, c["scale"], c["min_samples"])
    assert np.array_equal(vec[0], want[0]) and np.array_equal(vec[1], want[1])


def test_decluster_findings_in_the_reference():
    """What the kernel had wrong: cells 2^20 apart share the old 21-bit key, NaN rows belong to no cell
    and +-inf rows to their own (sorted last / first)."""
    cl = _reference()
    dxy, _ = cl.decluster(np.array([[3e6, 0.0], [902848.0, 0.0]]), np.arange(4.0).reshape(2, 2), 1)
    assert len(dxy) == 2
    assert (3_000_000 + 2 ** 20) % 2 ** 21 == (902_848 + 2 ** 20) % 2 ** 21
    coord = np.array([[1, 1], [np.nan, 2], [1, 2], [np.inf, 3], [np.inf, 5]], float)
    dxy, duv = cl.decluster(coord, np.arange(10.0).reshape(5, 2), 20)
    assert np.array_equal(dxy, [[1, 1.5], [np.inf, 4]]) and np.array_equal(duv, [[2, 3], [7, 8]])


def test_compaction_cases_are_what_they_claim():
    rng = np.random.default_rng(0)
    for tag, c in E.COMPACT.items():
        drop = E.compact_drop(c, rng)
        assert len(drop) == c["n"] and E.n_cap(c) >= c["n"], tag


def _overflows(xy, k):
    """queries (every row of xy against xy, min(k + 1, n) nearest) whose pending-node heap outgrows
    QHEAP on the host build of the device query"""
    from host_kernels import lib
    L = lib()
    L.host_kd_knn_pairs.restype = ctypes.c_int
    xy = np.ascontiguousarray(xy, dtype=np.float64)
    n = len(xy)
    kk = min(k + 1, n)
    perm = np.empty(n, np.int32)
    out = np.empty((n, kk), np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    return L.host_kd_knn_pairs(p(xy), n, p(xy), n, kk, -1, E.QHEAP, p(perm), p(out))


def _node_count(n):
    """an upper bound of the tree's node count, the one its node array is sized by (knn_body.cuh
    max_nodes): each query that spills takes this many arena entries at most"""
    return 2 * n + 1


def test_outlier_queries_stay_inside_the_spill_arena():
    """The device query moves a query whose pending-node heap outgrows QHEAP = 64 entries to a
    node-count-sized piece of a 2^17-entry arena, and traps when the arena runs out: the worst call of
    the grid must stay well inside ARENA / nnodes spills.  Stated margin: at most a quarter of it, with
    nnodes bounded by 2n + 1 (the grid's queries spill not at all today; 16000 points leave room for 4)."""
    worst = (0.0, "")
    for tag, c in E.KNN.items():
        xy, _ = E.knn_inputs(tag)
        if len(xy) < 2:
            continue
        spills = _overflows(xy, c["k"])
        room = E.ARENA // _node_count(len(xy))
        assert spills <= room // 4, (tag, spills, room)
        worst = max(worst, (spills / room, tag))
    assert worst[0] <= 0.25, worst
