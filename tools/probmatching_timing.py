"""Time probability matching (postprocessing.probmatching) at 2048^2, about half of the values exactly
0, float32 and float64: CUDA-event time of ``nonparam_match_empirical_cdf`` per call for device-tensor
and NumPy input (the whole call, read-backs and copies included), its two entry points' own kernels,
and ``resample_distributions`` split into the host draw, its upload and the kernels.  Medians of 20
calls.  Prints one JSON line per measurement, with the card, its power limit and SM clocks read in the
same run, and also writes them to $OUT/probmatching_timing.jsonl when OUT names a directory.

    python tools/probmatching_timing.py
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
from pysteps_b200.postprocessing import probmatching as pm  # noqa: E402
from probmatching_cases import rain  # noqa: E402

OUT = os.environ.get("OUT")
SIZE, REPS = 2048, 20
lines = []


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def call_ms(fn):
    """median CUDA-event time of whole calls, each ending in a synchronise"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(REPS):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def entry_ms(fn, entries):
    """median per call of the traced entry points' own time"""
    with _lib.Trace(only=entries) as tr:
        for _ in range(REPS):
            fn()
    summ = tr.summary()
    return {k: statistics.median(v) for k, v in summ.items()}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("probmatching_timing: no CUDA device")
    _device.require_cuda()
    emit(card=card())
    for dt in (np.float32, np.float64):
        name = np.dtype(dt).name
        for label, dry_x, dry_t in (("more_target", 0.55, 0.45), ("fewer_target", 0.45, 0.55)):
            x = rain((SIZE, SIZE), 1, dt, dry=dry_x)
            t = rain((SIZE, SIZE), 2, dt, dry=dry_t)
            dx, dtt = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
            ms_dev = call_ms(lambda: pm.nonparam_match_empirical_cdf(dx, dtt))
            ms_np = call_ms(lambda: pm.nonparam_match_empirical_cdf(x, t))
            k = entry_ms(lambda: pm.nonparam_match_empirical_cdf(dx, dtt), ("b200_pm_match_stats", "b200_pm_match"))
            emit(fn="nonparam_match_empirical_cdf", dtype=name, case=label, size=SIZE, tensor_ms=round(ms_dev, 3),
                 numpy_ms=round(ms_np, 3), **{f"{e}_ms": round(v, 3) for e, v in k.items()})

        a, b = rain((SIZE, SIZE), 3, dt), rain((SIZE, SIZE), 4, dt)
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        ms_dev = call_ms(lambda: pm.resample_distributions(da, db, 0.4))
        ms_np = call_ms(lambda: pm.resample_distributions(a, b, 0.4))
        k = entry_ms(lambda: pm.resample_distributions(da, db, 0.4), ("b200_pm_resample_nan", "b200_pm_resample"))
        draws = []
        for _ in range(REPS):
            t0 = time.perf_counter()
            d = np.random.binomial(1, 0.4, SIZE * SIZE).astype(bool)
            draws.append((time.perf_counter() - t0) * 1e3)
        up = call_ms(lambda: _device.to_device(d.view(np.uint8)))
        emit(fn="resample_distributions", dtype=name, size=SIZE, tensor_ms=round(ms_dev, 3), numpy_ms=round(ms_np, 3),
             host_draw_ms=round(statistics.median(draws), 3), draw_upload_ms=round(up, 3),
             **{f"{e}_ms": round(v, 3) for e, v in k.items()})
    emit(card_after=card())
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "probmatching_timing.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
