"""Time the DARTS motion method at 512^2, 2048^2 and 4096^2 (six seeded rain frames shifted by (3, -2) px
per step, the default keyword arguments): CUDA-event time of each device entry point
(b200_darts_spectrum, b200_darts_normal, b200_darts_synthesize; medians over 20 calls), a whole
motion.get_method("darts") call (host clock, NumPy input and device-tensor input; medians of 5), the
achieved FP64 rate of the spectrum from the operations its shapes require, and the reference's CPU
time where it can be imported (up to 2048^2).  Prints one JSON line per measurement, with the card,
its power limit and SM clocks read in the same run, and also writes them to $OUT/darts_timing.jsonl
when OUT names a directory.

    python tools/darts_timing.py
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
from pysteps_b200.motion import get_method  # noqa: E402

OUT = os.environ.get("OUT")
lines = []
ENTRIES = ("b200_darts_spectrum", "b200_darts_normal", "b200_darts_synthesize")


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def spectrum_flops(T, m, n, N_x=50, N_y=50, N_t=4, M_x=2, M_y=2):
    """FP64 operations of the three passes (a real x complex multiply-add is 4, complex x complex 8)"""
    K = N_x + M_x
    fx, Kx, Ky, Kt = min(K, n // 2) + 1, 2 * K + 1, 2 * (N_y + M_y) + 1, 2 * N_t + 1
    return 4 * T * m * n * fx + 8 * Kt * m * Kx * T + 8 * Kt * Ky * Kx * m


def main():
    if not torch.cuda.is_available():
        raise SystemExit("darts_timing: no CUDA device")
    _device.require_cuda()
    darts = get_method("darts")
    emit(card=card())
    ref = None
    try:
        import _refimport
        if _refimport.available():
            ref = _refimport.ref_module("pysteps.motion.darts")
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        emit(reference=f"not importable: {e}")
    for size in (512, 2048, 4096):
        R = syn.rain_frames(size, size, 6, seed=size + 1, dx=3, dy=-2)
        dR = torch.from_numpy(R).cuda()
        for _ in range(3):
            darts(dR, verbose=False)
        torch.cuda.synchronize()
        with _lib.Trace(only=ENTRIES) as tr:
            for _ in range(20):
                darts(dR, verbose=False)
        times = {k: statistics.median(v) for k, v in tr.summary().items()}
        flops = spectrum_flops(6, size, size)
        emit(size=size, T=6, kernel_ms={k.replace("b200_darts_", ""): round(v, 4) for k, v in times.items()},
             spectrum_gflop=round(flops / 1e9, 3),
             spectrum_fp64_tflops=round(flops / (times["b200_darts_spectrum"] * 1e-3) / 1e12, 3))
        for label, arg in (("device", dR), ("numpy", R)):
            ts = []
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = darts(arg, verbose=False)
                if isinstance(out, torch.Tensor):
                    torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            emit(size=size, T=6, input=label, whole_call_ms=round(statistics.median(ts), 3))
        if ref is not None and size <= 2048:
            t0 = time.perf_counter()
            want = ref.DARTS(R, verbose=False)
            tref = time.perf_counter() - t0
            got = darts(R, verbose=False)
            emit(size=size, T=6, reference_cpu_s=round(tref, 3),
                 max_rel_diff=float(np.abs(got - want).max() / np.abs(want).max()))
        else:
            emit(size=size, T=6, reference_cpu_s="not measured")
    emit(card_after=card())
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "darts_timing.jsonl"), "w") as f:
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
