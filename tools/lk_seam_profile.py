"""The seam between the sparse LK stages and the advection in bench.py's headline step (2048^2, dense
LK + 12 leadtimes, device-resident, seeded bench.make_inputs), under torch.profiler.

    python tools/lk_seam_profile.py OUTDIR [--steps 20] [--warmup 5]

Writes OUTDIR/lk_seam_trace.json (Chrome trace), OUTDIR/lk_seam_kernels.json and OUTDIR/lk_seam.md, and
prints the table:
  - every kernel (and memset / copy) between the end of decluster_kernel and the start of the trajectory
    kernel, mean per step: what b200_idw_fill (or the plan + planned fill) costs, kernel by kernel
  - the idle time on the main stream between the end of decluster_kernel and the start of the first fill
    kernel (idw32_kernel / idw_kernel / idw_plan_const_kernel): the gap the GPU waits for the host
  - the re-layout of the field before the trajectory kernel (relayout_kernel)
The L2 is flushed between steps as in bench.py (outside the steps).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FILL_FIRST = ("idw32_kernel", "idw_kernel", "idw_plan_const_kernel")
RELAYOUT = ("relayout_kernel",)


def _short(name):
    """kernel name without namespace / template arguments / parameter list (names in an anonymous
    namespace start with "(anonymous namespace)::")"""
    base = name.replace("(anonymous namespace)::", "").split("(")[0]
    for tok in ("idw32_kernel", "idw_kernel", "idw_plan_const_kernel", "idw_plan_kernel", "kd_build_kernel",
                "kd_build_serial_kernel", "idw_fix_warp_kernel", "idw_fix_kernel", "decluster_kernel",
                "relayout_kernel", "sl_multistep_kernel"):
        if tok in base:
            tmpl = base[base.find("<"):base.find(">") + 1] if "<" in base and tok == "idw_kernel" else ""
            return tok + tmpl
    return base[:80]


def _union(iv):
    tot, end = 0.0, -1e300
    for a, b in sorted(iv):
        if b <= end:
            continue
        tot += b - max(a, end)
        end = b
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.outdir, exist_ok=True)

    import bench
    import pysteps_b200
    w = bench.WORKLOADS["lk_sl12_2048"]
    frames_h, precip_h, _ = bench.make_inputs(w, 0)
    frames = torch.from_numpy(frames_h).cuda()
    precip = torch.from_numpy(precip_h).cuda()
    lk = pysteps_b200.motion.get_method("lk")
    extrap = pysteps_b200.extrapolation.get_method("semilagrangian")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def step():
        V = lk(frames)
        return extrap(precip, V, w["T"])

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            flush.fill_(1)
            torch.cuda.synchronize()
            step()
            torch.cuda.synchronize()
    trace_path = os.path.join(args.outdir, "lk_seam_trace.json")
    prof.export_chrome_trace(trace_path)
    with open(trace_path) as f:
        tr = json.load(f)
    ev = tr["traceEvents"] if isinstance(tr, dict) else tr
    gpu = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    gpu.sort(key=lambda e: e["ts"])
    decl = [e for e in gpu if "decluster_kernel" in e["name"]]
    sl = [e for e in gpu if "sl_multistep_kernel" in e["name"]]
    assert len(decl) == args.steps, f"{len(decl)} decluster launches in {args.steps} steps"
    main_stream = decl[0]["args"].get("stream")
    per = {}
    gaps, waits, relayout = [], [], []
    for d in decl:
        d_end = d["ts"] + d["dur"]
        s_start = min(e["ts"] for e in sl if e["ts"] > d_end)
        seam = [e for e in gpu if d_end <= e["ts"] < s_start]
        for e in seam:
            key = (e["cat"], _short(e["name"]))
            per.setdefault(key, []).append(e["dur"])
        first = min((e["ts"] for e in seam if e["cat"] == "kernel" and _short(e["name"]).split("<")[0] in FILL_FIRST),
                    default=None)
        if first is not None:
            busy = [(max(e["ts"], d_end), min(e["ts"] + e["dur"], first)) for e in seam
                    if e["args"].get("stream") == main_stream and e["ts"] < first]
            gaps.append((first - d_end) - _union(busy))
            waits.append(first - d_end)
        relayout.append(sum(e["dur"] for e in seam if _short(e["name"]) in RELAYOUT))
    n = args.steps
    assert gaps, "no fill kernel found after decluster_kernel"
    rows = sorted(({"cat": c, "name": k, "calls_per_step": len(v) / n, "us_per_step": sum(v) / n}
                   for (c, k), v in per.items()), key=lambda r: -r["us_per_step"])
    res = {"steps": n, "device": torch.cuda.get_device_name(0),
           "idle_gap_us": {"mean": float(np.mean(gaps)), "median": float(np.median(gaps)),
                           "min": float(np.min(gaps)), "max": float(np.max(gaps))},
           "decluster_end_to_first_fill_kernel_us": float(np.mean(waits)),
           "relayout_us_per_step": float(np.mean(relayout)),
           "seam_ops": rows}
    with open(os.path.join(args.outdir, "lk_seam_kernels.json"), "w") as f:
        json.dump(res, f, indent=1)
    lines = [f"# LK seam, {res['device']}, {n} steps (mean per step)", "",
             f"idle gap on the main stream, decluster end -> first fill kernel: mean {res['idle_gap_us']['mean']:.1f} us "
             f"(median {res['idle_gap_us']['median']:.1f}, min {res['idle_gap_us']['min']:.1f}, max {res['idle_gap_us']['max']:.1f})",
             f"decluster end -> first fill kernel start: {res['decluster_end_to_first_fill_kernel_us']:.1f} us",
             f"re-layout of the field (interleave / widen): {res['relayout_us_per_step']:.1f} us", "",
             "| op | name | calls/step | us/step |", "|---|---|---|---|"]
    lines += [f"| {r['cat']} | `{r['name']}` | {r['calls_per_step']:.2f} | {r['us_per_step']:.1f} |" for r in rows]
    text = "\n".join(lines) + "\n"
    with open(os.path.join(args.outdir, "lk_seam.md"), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
