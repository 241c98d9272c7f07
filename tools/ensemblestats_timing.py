"""Time the ensemble statistics (postprocessing.get_method(..., "ensemblestats")) at 24 members x 2048^2,
about half of the values exactly 0, float32 and float64, device-tensor input: CUDA-event time of
``mean``, ``excprob`` with 1 and with 4 thresholds (medians of 20 calls, each call's own kernels
traced), the bytes each reduction moves (X read once, the output written once) over its kernel time,
against the H100's 3.35 TB/s; and ``banddepth`` split into the mask kernels, the host draw of the
random tie-breaks, their upload and the rank kernel.  Prints one JSON line per measurement, with the
card, its power limit and SM clocks read in the same run, and also writes them to
$OUT/ensemblestats_timing.jsonl when OUT names a directory.

    python tools/ensemblestats_timing.py
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
from pysteps_b200.postprocessing import get_method  # noqa: E402
from ensemblestats_cases import rain  # noqa: E402

OUT = os.environ.get("OUT")
K, SIZE, HBM = 24, 2048, 3.35e12
lines = []


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def kernel_ms(fn, entry, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with _lib.Trace(only=(entry,)) as tr:
        for _ in range(reps):
            fn()
    return statistics.median(tr.summary()[entry])


def main():
    if not torch.cuda.is_available():
        raise SystemExit("ensemblestats_timing: no CUDA device")
    _device.require_cuda()
    emit(card=card())
    mean, excprob, banddepth = (get_method(n, "ensemblestats") for n in ("mean", "excprob", "banddepth"))
    N = SIZE * SIZE
    for dt in (np.float32, np.float64):
        X = rain(K, (SIZE, SIZE), 71, dt)
        d = torch.from_numpy(X).cuda()
        size = np.dtype(dt).itemsize
        for label, fn, entry, out_bytes in (
                ("mean", lambda: mean(d), "b200_ensemble_mean", size),
                ("mean_ignore_nan", lambda: mean(d, ignore_nan=True), "b200_ensemble_mean", size),
                ("excprob_1", lambda: excprob(d, 0.5), "b200_ensemble_excprob", 8),
                ("excprob_4", lambda: excprob(d, [0.1, 0.5, 1.0, 5.0]), "b200_ensemble_excprob", 32)):
            ms = kernel_ms(fn, entry)
            nbytes = K * N * size + N * out_bytes
            emit(dtype=np.dtype(dt).name, members=K, size=SIZE, call=label, kernel_ms=round(ms, 4),
                 gb=round(nbytes / 1e9, 3), tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 2),
                 of_hbm_peak=round(nbytes / (ms * 1e-3) / HBM, 3))
            ts = []
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            emit(dtype=np.dtype(dt).name, call=label, whole_call_ms=round(statistics.median(ts), 3))
        # banddepth: the mask kernels, the host draw, the upload and the rank kernel
        np.random.seed(0)
        banddepth(d)
        torch.cuda.synchronize()
        with _lib.Trace(only=("b200_ensemble_band_mask", "b200_ensemble_band_match")) as tr:
            t0 = time.perf_counter()
            banddepth(d)
            torch.cuda.synchronize()
            whole = (time.perf_counter() - t0) * 1e3
        dev = {k: v[0] for k, v in tr.summary().items()}
        p = int((np.isfinite(X).all(axis=0) & (X >= np.nanmin(X)).any(axis=0)).sum())  # the masked pixels
        t0 = time.perf_counter()
        b = np.random.random((K, p))
        draw = (time.perf_counter() - t0) * 1e3
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        _device.to_device(b)
        end.record()
        torch.cuda.synchronize()
        emit(dtype=np.dtype(dt).name, members=K, size=SIZE, call="banddepth", p=p,
             mask_ms=round(dev["b200_ensemble_band_mask"], 4), host_draw_ms=round(draw, 2),
             upload_ms=round(start.elapsed_time(end), 3), upload_gb=round(b.nbytes / 1e9, 3),
             rank_ms=round(dev["b200_ensemble_band_match"], 3), whole_call_ms=round(whole, 2))
        del d
        torch.cuda.empty_cache()
    emit(card_after=card())
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "ensemblestats_timing.jsonl"), "w") as f:
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
