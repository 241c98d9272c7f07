"""Time linear and salient blending (blending.get_method("linear_blending" | "salient_blending")) at 24 NWP
members x 2048^2, T = 12 (timestep 5, window 15..45 min: 5 leads inside it), float32 NWP, device-tensor
input: CUDA-event time of the extrapolation nowcast, the conversion of the nowcast and of the NWP
("dB" and mm/h), the dense rank of one 24 x 2048^2 slab (sort and rank, b200_dense_rank), the blend
kernels (b200_blend_linear, b200_blend_salient per lead) and whole calls (medians of 5).  The linear
kernel's compulsory bytes (the NWP read once, the output written once, the nowcast once per lead) are rated
against the H100's 3.35 TB/s.  The reference's own CPU time at 512^2 (3 NWP members) where it can be
imported.  One JSON line per measurement, with the card, its power limit and SM clocks read in the same
run; also written to $OUT/blending_timing.jsonl when OUT names a directory.

    python tools/blending_timing.py
"""
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "golden")]
from pysteps_b200 import _device, _lib  # noqa: E402
from pysteps_b200.blending import get_method  # noqa: E402
from pysteps_b200.blending.linear_blending import to_rainrate  # noqa: E402
from pysteps_b200.nowcasts import get_method as nowcast  # noqa: E402

OUT = os.environ.get("OUT")
E, T, SIZE, HBM = 24, 12, 2048, 3.35e12
KW = dict(start_blending=15, end_blending=45)
MM = {"unit": "mm/h", "transform": None}
lines = []


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, smax, sm = [x.strip() for x in r.stdout.strip().split("\n")[0].split(",")]
    return dict(card=name, power_limit=power, sm_clock_max=smax, sm_clock=sm)


def timed(fn, reps=5):
    out = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e))
    return statistics.median(out)


def traced(fn, names):
    with _lib.Trace(only=names) as tr:
        fn()
        got = tr.summary()
    return {k: sum(v) for k, v in got.items()}


def main():
    _device.require_cuda()
    c = card()
    rng = np.random.default_rng(0)
    P = torch.from_numpy(rng.gamma(0.8, 2.0, (SIZE, SIZE))).cuda()
    R = torch.from_numpy(rng.gamma(0.8, 2.0, (E, T, SIZE, SIZE)).astype(np.float32)).cuda()
    V = torch.from_numpy(rng.uniform(-3, 3, (2, SIZE, SIZE))).cuda()
    f_now = nowcast("extrapolation")
    f_now(P, V, 9)
    emit(what="extrapolation nowcast, 2048^2 float64, 9 leads", ms=timed(lambda: f_now(P, V, 9)), **c)
    dbP = torch.from_numpy(10 * np.log10(rng.gamma(0.8, 2.0, (9, SIZE, SIZE)) + 0.01)).cuda()
    to_rainrate(dbP, {"unit": "mm/h", "transform": "dB", "threshold": -10.0})
    emit(what="conversion dB -> mm/h of the 9-lead float64 nowcast",
         ms=timed(lambda: to_rainrate(dbP, {"unit": "mm/h", "transform": "dB", "threshold": -10.0})), **c)
    Rmm = {"unit": "mm", "transform": None, "accutime": 5, "threshold": 0.1, "zerovalue": 0.0}
    emit(what="conversion mm -> mm/h of the 24 x 12 float32 NWP", ms=timed(lambda: to_rainrate(R, Rmm)), **c)

    n = E * SIZE * SIZE
    x = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).cuda()
    nb = _lib.c_i64(0)
    _lib.call("b200_blend_scratch_bytes", n, ctypes.byref(nb))
    scratch = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    rank = torch.empty(n, dtype=torch.int32, device="cuda")
    info = torch.zeros(2, dtype=torch.int32, device="cuda")

    def rank_once():
        _lib.call("b200_dense_rank", x.data_ptr(), _lib.F32, n, rank.data_ptr(), info[0:1].data_ptr(),
                  info[1:2].data_ptr(), scratch.data_ptr(), nb.value, _device.stream_ptr())
    rank_once()
    emit(what="dense rank (radix sort + rank scan) of one 24 x 2048^2 float32-valued slab", ms=timed(rank_once),
         scratch_bytes=nb.value, **c)

    for name in ("linear_blending", "salient_blending"):
        f = get_method(name)

        def call():
            return f(P, MM, V, T, 5, "extrapolation", R, MM, **KW)
        call()
        torch.cuda.synchronize()
        emit(what=f"{name}: whole call, device tensors", ms=timed(call, 3), **c)
        k = traced(call, {"b200_blend_linear", "b200_blend_salient"})
        row = dict(what=f"{name}: blend kernels (one call)", ms={a: round(b, 3) for a, b in k.items()}, **c)
        if "b200_blend_linear" in k:
            # compulsory traffic: every NWP value read once and every output value written once (float32), and
            # the nowcast's (float64) planes once per lead it is read in (the 24 members re-read it from L2)
            lin_leads = 12 if name == "linear_blending" else 12 - 5
            now_leads = 9 if name == "linear_blending" else 9 - 5
            b = E * lin_leads * SIZE * SIZE * (4 + 4) + now_leads * SIZE * SIZE * 8
            row.update(linear_bytes=b, linear_tb_s=b / (k["b200_blend_linear"] * 1e-3) / 1e12, hbm_tb_s=HBM / 1e12)
        emit(**row)

    try:
        import _refimport
        if _refimport.available():
            lb = _refimport.ref_module("pysteps.blending.linear_blending")
            p = rng.gamma(0.8, 2.0, (512, 512))
            r = rng.gamma(0.8, 2.0, (3, T, 512, 512))
            for sal in (False, True):
                t0 = time.perf_counter()
                lb.forecast(p, MM, np.zeros((2, 512, 512)), T, 5, "eulerian", r, MM, saliency=sal, **KW)
                emit(what=f"reference CPU, 512^2, 3 members, saliency={sal}", s=time.perf_counter() - t0,
                     cpu_count=os.cpu_count())
    except Exception as e:  # noqa: BLE001 -- the reference is optional here
        emit(what="reference CPU", skipped=repr(e))
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "blending_timing.jsonl"), "w") as fh:
            fh.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
