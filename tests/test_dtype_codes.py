"""CPU test of the dtype-code rule of include/pysteps_b200.h: every entry point that takes a field dtype
code refuses a code other than B200_F32 / B200_F64 with B200_EINVAL, and names it, before any device
work and before any early return on empty input.  The semi-Lagrangian row, trajectory, batched,
interleave and BPS entries are covered by test_capi.py.

The calls run in a child process that sees no CUDA device, with every other argument valid and
placeholder device pointers: an entry point that slipped past its check would fail with a CUDA
"no device" code, or return 0 on an empty call, and never touch a GPU."""
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = 100001
BAD_CODES = (2, -1)
# entry points whose refusals test_capi.py checks
IN_TEST_CAPI = {"b200_sl_extrapolate_rows", "b200_sl_extrapolate_rows_f32", "b200_sl_trajectories",
                "b200_sl_step_batched", "b200_sl_interleave_velocity", "b200_bps_perturb_velocity"}


def _cases():
    """(entry point, arguments in order, dtype groups, overrides of an empty call or None, extra overrides).
    A group (what, name) is one code taken by with_dtype; (what, a, b) a pair taken by with_dtypes."""
    from pysteps_b200 import _lib
    buf = 0x1000  # a device pointer that is never dereferenced
    big = 1 << 40  # scratch_bytes beyond any carve of these sizes

    def host(values, ctype):
        a = np.ascontiguousarray(values, dtype={ctypes.c_double: np.float64, ctypes.c_int: np.int32,
                                                ctypes.c_int64: np.int64}[ctype])
        return a.ctypes.data_as(ctypes.POINTER(ctype)), a  # the array keeps the memory alive

    keep = []

    def h(values, ctype=ctypes.c_double):
        p, a = host(values, ctype)
        keep.append(a)
        return p

    m, n, T, k, N = 8, 8, 2, 3, 64
    sl = dict(precip=buf, velocity=buf, xy=None, disp_prev=None, tdiff=h(np.ones(4)), T=4, vts=1.0, n_iter=1,
              outval=0.0, mode=0, vdt=1, layout=0, pdt=1, m=m, n=n, out=buf, disp_out=None, stream=None)
    sl_host = dict(precip=h(np.zeros(m * n)), velocity=h(np.zeros(2 * m * n)), xy=None, disp_prev=None,
                   tdiff=h(np.ones(4)), T=4, vts=1.0, n_iter=1, outval=0.0, mode=0, vdt=1, pdt=1, m=m, n=n,
                   out=h(np.zeros(4 * m * n)), disp_out=None)
    pair_fo, pair_po = ("field", "f_dt", "o_dt"), ("field", "p_dt", "o_dt")
    cases = [
        ("b200_sl_extrapolate", sl, [("field", "vdt", "pdt")], None),
        ("b200_sl_extrapolate_host", sl_host, [("field", "vdt", "pdt")], None),
        ("b200_spline_prepare",
         dict(precip=buf, pdt=1, m=m, n=n, order=3, mode=0, stats=buf, zero_fill=0, poles=h([3 ** 0.5 - 2]),
              zpow0=h([0.01]), zpow1=h([0.01]), coeffs=buf, mask_min=buf, mask_finite=buf, stream=None),
         [("precip", "pdt")], None),
        ("b200_spline_sample",
         dict(coeffs=buf, m=m, n=n, order=3, mode=0, xy=None, disp_steps=buf, T=T, row_begin=0, row_count=m,
              outval=0.0, mask_min=buf, mask_finite=buf, stats=buf, odt=1, out=buf, stream=None),
         [("output", "odt")], None),
        ("b200_proesmans_scale",
         dict(frames=buf, dt=1, count=N, im_min=0.0, im_max=1.0, do_scale=1, out=buf, stream=None),
         [("frame", "dt")], None),
        ("b200_field_stats", dict(a=buf, dt=1, count=N, stats=buf, stream=None), [("field", "dt")], dict(count=0)),
        ("b200_constant_eval",
         dict(prev=buf, next=buf, dt=1, m=m, n=n, vx=0.5, vy=0.5, scratch=buf, record=buf, stream=None),
         [("frame", "dt")], dict(m=0)),
        ("b200_darts_spectrum",
         dict(frames=buf, dt=1, T=T, m=m, n=n, tw_x=buf, fx=5, tw_y=buf, Ky=3, tw_t=buf, Kt=3, K=1, work=buf,
              spectrum=buf, stream=None),
         [("frame", "dt")], None),
        ("b200_probability",
         dict(field=buf, dt=1, plane_stride=m * n, T=T, m=m, n=n, threshold=0.5, nan_exceeds=0,
              scales=h([0, 3], ctypes.c_int), runs=buf, scratch=buf, out=buf, stream=None),
         [("field", "dt")], dict(T=0)),
        ("b200_ensemble_mean",
         dict(X=buf, dt=1, k=k, N=N, nan_mode=1, use_thr=1, thr=0.1, out=buf, flags=buf, stream=None),
         [("field", "dt")], dict(N=0)),
        ("b200_ensemble_excprob",
         dict(X=buf, dt=1, k=k, N=N, thr=h([0.1, 1.0]), n_thr=2, ignore_nan=0, out=buf, flags=buf, stream=None),
         [("field", "dt")], dict(N=0)),
        ("b200_ensemble_band_mask", dict(X=buf, dt=1, k=k, N=N, thr=0.1, col=buf, p=buf, stream=None),
         [("field", "dt")], dict(N=0)),
        ("b200_ensemble_band_match", dict(X=buf, dt=1, k=k, N=N, col=buf, b=buf, p=4, match=buf, stream=None),
         [("field", "dt")], dict(N=0, p=0)),
        ("b200_blend_transform",
         dict(x=buf, y=buf, dt=1, n=N, kind=4, lam=0.5, thr=0.1, zero=0.0, fix_idx=buf, fix_x=buf, cap=8,
              nfix=buf, stream=None),
         [("field", "dt")], dict(n=0)),
        ("b200_blend_unit", dict(x=buf, y=buf, dt=1, n=N, kind=1, a=1.0, b=2.0, stream=None), [("field", "dt")],
         dict(n=0)),
        ("b200_blend_scatter", dict(y=buf, dt=1, idx=buf, val=buf, n=N, stream=None), [("field", "dt")],
         dict(n=0)),
        ("b200_blend_linear",
         dict(now=buf, now_dt=0, now_map=buf, now_member=T * N, nwp=buf, nwp_dt=0, nwp_map=buf, nwp_member=T * N,
              out=buf, n_out=2, T=T, P=N, mode=buf, bits=buf, w_nwp=buf, w_now=buf, fill_nwp=1, stream=None),
         [("field", "now_dt", "nwp_dt")], dict(P=0), [dict(now_dt=2, nwp_dt=-1)]),
        ("b200_blend_salient",
         dict(now=buf, now_dt=0, now_map=buf, now_member=T * N, nwp=buf, nwp_dt=0, nwp_map=buf, nwp_member=T * N,
              out=buf, n_out=2, T=T, P=N, lead=0, w=0.5, w1=0.5, w2=0.25, w12=0.25, fill_nwp=1, scratch=buf,
              scratch_bytes=big, stream=None),
         [("field", "now_dt", "nwp_dt")], dict(P=0), [dict(now_dt=2, nwp_dt=-1)]),
        ("b200_dense_rank",
         dict(x=buf, dt=1, n=N, rank=buf, max_rank=buf, nan_flag=buf, scratch=buf, scratch_bytes=big, stream=None),
         [("field", "dt")], dict(n=0)),
        ("b200_pairwise_sum",
         dict(x=buf, dt=1, seg_off=h([0], ctypes.c_int64), seg_len=h([N], ctypes.c_int64), nseg=1, out=buf,
              stream=None),
         [("field", "dt")], dict(nseg=0)),
        ("b200_verif_crps", dict(Xf=buf, f_dt=1, Xo=buf, o_dt=1, k=k, N=N, res=buf, n=buf, stream=None),
         [pair_fo], dict(N=0)),
        ("b200_verif_rankhist",
         dict(Xf=buf, f_dt=1, Xo=buf, o_dt=1, k=k, N=N, use_min=1, thr_f=0.1, sub_f=0.0, thr_o=0.1, sub_o=0.0,
              hist=buf, ties=buf, n_ties=buf, stream=None),
         [pair_fo], dict(N=0)),
        ("b200_verif_reldiag",
         dict(P=buf, p_dt=1, Xo=buf, o_dt=1, N=N, edges=h([0.0, 0.5, 1.0]), n_edges=3, thr_o=0.1, sorted=buf,
              seg=buf, above=buf, stream=None),
         [pair_po], dict(N=0)),
        ("b200_verif_roc",
         dict(P=buf, p_dt=1, Xo=buf, o_dt=1, N=N, thr=h([0.25, 0.75]), n_thr=2, thr_o=0.1, counts=buf,
              stream=None),
         [pair_po], dict(N=0)),
        ("b200_verif_contab",
         dict(pred=buf, p_dt=1, obs=buf, o_dt=1, thr_p=0.1, thr_o=0.1, kept_size=h([4], ctypes.c_int64),
              kept_stride=h([16], ctypes.c_int64), n_kept=1, red_size=h([16], ctypes.c_int64),
              red_stride=h([1], ctypes.c_int64), n_red=1, counts=buf, stream=None),
         [pair_po], None),
        ("b200_verif_cont_moments",
         dict(pred=buf, p_dt=1, obs=buf, o_dt=1, conditioning=1, thr_p=0.1, thr_o=0.1,
              kept_size=h([4], ctypes.c_int64), kept_stride=h([16], ctypes.c_int64), n_kept=1, outer_size=None,
              outer_stride=None, n_outer=0, L=16, tot=buf, cnt=buf, infs=buf, flags=buf, stream=None),
         [pair_po], None),
        ("b200_fss_fractions",
         dict(X=buf, dt=1, nf=2, m=m, n=n, thr=0.1, sub=0.0, s=3, S=buf, stream=None), [("field", "dt")],
         dict(nf=0)),
        ("b200_pm_match_stats",
         dict(x=buf, x_dt=1, ignore=None, n_x=N, t=buf, t_dt=1, n_t=N, stats=buf, scratch=buf, scratch_bytes=big,
              stream=None),
         [("field", "x_dt", "t_dt")], dict(n_x=0, n_t=0)),
        ("b200_pm_match",
         dict(x=buf, x_dt=1, ignore=None, t=buf, t_dt=1, n=N, stats=buf, n_xwet=10, n_twet=20, clip=1, i0=2, i1=3,
              gamma=0.5, out=buf, scratch=buf, scratch_bytes=big, stream=None),
         [("field", "x_dt", "t_dt")], dict(n=0, n_xwet=0, n_twet=0, clip=0)),
        ("b200_pm_resample_nan", dict(a=buf, a_dt=1, b=buf, b_dt=1, n=N, n_nan=buf, stream=None),
         [("field", "a_dt", "b_dt")],
         dict(n=0)),
        ("b200_pm_resample",
         dict(a=buf, a_dt=1, b=buf, b_dt=1, n=N, n_nan=2, draws=buf, out=buf, out_dt=1, scratch=buf,
              scratch_bytes=big, stream=None),
         [("field", "a_dt", "b_dt"), ("output", "out_dt")], dict(n=0, n_nan=0)),
    ]
    out = []
    for case in cases:
        fn, args, groups, empty = case[:4]
        extra = case[4] if len(case) > 4 else []
        assert len(args) == len(_lib._SIGNATURES[fn][1]), fn
        calls = [{name: bad} for g in groups for name in g[1:] for bad in BAD_CODES] + extra
        calls += [dict(c, **empty) for c in calls[:1] if empty is not None]
        for kw in calls:
            out.append((fn, args, groups, kw))
    return out, keep


def _expected(groups, args):
    for what, *names in groups:
        codes = [args[name] for name in names]
        if any(c not in (0, 1) for c in codes):
            return f"unknown {what} dtype {codes[0]}" if len(codes) == 1 else \
                f"unknown {what} dtypes {codes[0]} / {codes[1]}"
    raise AssertionError("no unknown code")


def _child():
    """Run every refused call and print one JSON record per call."""
    from pysteps_b200 import _lib
    lib = _lib.load()
    cases, _keep = _cases()
    records = []
    for fn, defaults, groups, kw in cases:
        args = dict(defaults, **kw)
        rc = getattr(lib, fn)(*args.values())
        records.append(dict(fn=fn, kw=kw, rc=rc, msg=lib.b200_last_error().decode(), want=_expected(groups, args)))
    print(json.dumps(records))


def _header_entry_points_with_dtypes():
    from pysteps_b200 import _lib
    with open(_lib.HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return {m.group(1) for m in re.finditer(r"\b(b200_[a-z0-9_]+)\s*\(([^)]*)\)", text)
            if re.search(r"\bint\s+\w*dtype\b", m.group(2))}


def test_unknown_dtype_codes_are_refused_before_device_work():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    r = subprocess.run([sys.executable, "-c", "import test_dtype_codes; test_dtype_codes._child()"], env=env,
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    records = json.loads(r.stdout.strip().splitlines()[-1])
    assert {rec["fn"] for rec in records} == _header_entry_points_with_dtypes() - IN_TEST_CAPI
    bad = [(rec["fn"], rec["kw"], rec["rc"], rec["msg"]) for rec in records
           if (rec["rc"], rec["msg"]) != (EINVAL, rec["want"])]
    assert not bad, "\n".join(map(str, bad))
