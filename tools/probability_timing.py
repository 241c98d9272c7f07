"""Time the local Lagrangian probability nowcast (nowcasts.get_method("probability")) at 2048^2, T = 12,
slope 5, threshold 5 (a seeded rain field with a NaN disc, a smooth advection field): CUDA-event time
of the neighbourhood step alone (b200_probability: 12 prefix and 12 ratio kernels; median of 20
calls) and of the extrapolation it follows, a whole call (host clock, NumPy input and device-tensor
input; medians of 5), the prefix loads the ratio kernels make (two 8-byte words per kernel row that
overlaps the frame, per pixel), and the reference's CPU time at 1024^2 where it can be imported.
Prints one JSON line per measurement, with the card, its power limit and SM clocks read in the same
run, and also writes them to $OUT/probability_timing.jsonl when OUT names a directory.

    python tools/probability_timing.py
"""
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
from pysteps_b200 import _synthetic as syn  # noqa: E402
from pysteps_b200.nowcasts import get_method  # noqa: E402

OUT = os.environ.get("OUT")
lines = []
T, SLOPE, THR = 12, 5, 5.0


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def prefix_bytes(m, n):
    """8-byte prefix words the ratio kernels read: two per overlapping kernel row per pixel"""
    total = 0
    for t in range(1, T + 1):
        s, c = int(t * SLOPE), (int(t * SLOPE) - 1) // 2
        y = np.arange(m)
        rows = np.minimum(s - 1, y + c) - np.maximum(0, y + c - (m - 1)) + 1
        total += 2 * 8 * n * int(rows.sum())
    return total


def inputs(size, seed):
    P = syn.nan_disc(syn.rain_field(size, size, seed), 0.1)
    return P, syn.velocity_field(size, size, seed)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("probability_timing: no CUDA device")
    _device.require_cuda()
    fc = get_method("probability")
    emit(card=card())
    size = 2048
    P, V = inputs(size, 31)
    dP, dV = torch.from_numpy(P).cuda(), torch.from_numpy(V).cuda()
    for _ in range(3):
        fc(dP, dV, T, THR, slope=SLOPE)
    torch.cuda.synchronize()
    with _lib.Trace(only=("b200_probability", "b200_sl_extrapolate_rows")) as tr:
        for _ in range(20):
            fc(dP, dV, T, THR, slope=SLOPE)
    times = {k: statistics.median(v) for k, v in tr.summary().items()}
    nbytes = prefix_bytes(size, size)
    emit(size=size, T=T, slope=SLOPE, neighbourhood_ms=round(times["b200_probability"], 4),
         extrapolation_ms=round(times["b200_sl_extrapolate_rows"], 4),
         prefix_gb=round(nbytes / 1e9, 2),
         prefix_tb_per_s=round(nbytes / (times["b200_probability"] * 1e-3) / 1e12, 2))
    for label, args in (("device", (dP, dV)), ("numpy", (P, V))):
        ts = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fc(*args, T, THR, slope=SLOPE)
            if isinstance(out, torch.Tensor):
                torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        emit(size=size, T=T, input=label, whole_call_ms=round(statistics.median(ts), 3))
    ref = None
    try:
        import _refimport
        if _refimport.available():
            ref = _refimport.ref_module("pysteps.nowcasts.lagrangian_probability")
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        emit(reference=f"not importable: {e}")
    if ref is not None:
        P1, V1 = inputs(1024, 32)
        t0 = time.perf_counter()
        want = ref.forecast(P1, V1, T, THR, slope=SLOPE)
        tref = time.perf_counter() - t0
        got = fc(P1, V1, T, THR, slope=SLOPE)
        nan = np.isnan(want)
        emit(size=1024, T=T, reference_cpu_s=round(tref, 3), same_nan=bool(np.array_equal(nan, np.isnan(got))),
             max_abs_diff=float(np.abs(got[~nan] - want[~nan]).max()))
    else:
        emit(size=1024, T=T, reference_cpu_s="not measured")
    emit(card_after=card())
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "probability_timing.jsonl"), "w") as f:
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
