"""Time the verification scores (pysteps_b200.verification) at 24 members x 2048^2, rain with about
60 % exact zeros, float32 and float64, NumPy and device-tensor input: the wall time of a whole
CRPS_accum, rankhist_accum, reldiag_accum and ROC_curve_accum call (medians of 5, synchronised), the
CUDA-event time of each score's kernels (medians of 5 calls, every C-ABI call traced), and for
rankhist the host draw of the tie-breaks and their upload apart; CRPS at 300 members x 1024^2; then the reference's time for the
same calls on this machine's CPU where the reference can be imported (one run each).  Prints one JSON
line per measurement, with the card, its power limit and SM clocks read in the same run, and also
writes them to $OUT/verification_timing.jsonl when OUT names a directory.

    python tools/verification_timing.py [--no-reference]
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tests")]
from pysteps_b200 import _device, _lib  # noqa: E402
from pysteps_b200.verification import ensscores, probscores  # noqa: E402
from verification_cases import rain, reference  # noqa: E402

OUT = os.environ.get("OUT")
K, SIZE = 24, 2048
lines = []


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def wall_ms(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t)


def traced_ms(fn, reps=5):
    """median over calls of the summed kernel time of every C-ABI entry point"""
    fn()
    torch.cuda.synchronize()
    per = {}
    for _ in range(reps):
        with _lib.Trace() as tr:
            fn()
        for name, v in tr.summary().items():
            per.setdefault(name, []).append(sum(v))
    return {name: round(statistics.median(v), 4) for name, v in per.items()}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("verification_timing: no CUDA device")
    _device.require_cuda()
    emit(card=card())
    rng = np.random.default_rng(0)
    for dt in (np.float32, np.float64):
        X_f = rain(rng, (K, SIZE, SIZE), dt, zeros=0.6)
        X_o = rain(rng, (SIZE, SIZE), dt, zeros=0.6)
        P = (X_f >= 1.0).mean(axis=0).astype(dt)
        for kind in ("numpy", "tensor"):
            f, o, p = (X_f, X_o, P) if kind == "numpy" else \
                (torch.from_numpy(X_f).cuda(), torch.from_numpy(X_o).cuda(), torch.from_numpy(P).cuda())
            calls = {
                "CRPS": lambda: probscores.CRPS_accum(probscores.CRPS_init(), f, o),
                "rankhist": lambda: ensscores.rankhist_accum(ensscores.rankhist_init(K, 0.1), f, o),
                "reldiag": lambda: probscores.reldiag_accum(probscores.reldiag_init(1.0), p, o),
                "ROC": lambda: probscores.ROC_curve_accum(probscores.ROC_curve_init(1.0), p, o),
            }
            for name, fn in calls.items():
                emit(score=name, dtype=np.dtype(dt).name, input=kind, members=K, size=SIZE, call_ms=round(wall_ms(fn), 3),
                     kernels_ms=traced_ms(fn) if kind == "tensor" else None)
        # the tie-breaks of rankhist: how many, their host draw and their upload
        counts = ensscores.rankhist_init(K, 0.1)
        h = torch.empty(K + 1, dtype=torch.int64, device="cuda")
        ties = torch.empty((SIZE * SIZE, 2), dtype=torch.int32, device="cuda")
        d_n = torch.empty(1, dtype=torch.int64, device="cuda")
        f = torch.from_numpy(X_f).cuda().reshape(K, -1)
        o = torch.from_numpy(X_o).cuda().reshape(-1)
        code = _device.dtype_code(f.dtype)
        sub = float(np.asarray(0.1 - 1).astype(dt))
        thr = float(np.asarray(0.1).astype(dt))
        _lib.call("b200_verif_rankhist", f.data_ptr(), code, o.data_ptr(), code, K, SIZE * SIZE, 1, thr, sub, thr, sub,
                  h.data_ptr(), ties.data_ptr(), d_n.data_ptr(), _device.stream_ptr())
        n_ties = int(_device.to_host(d_n)[0])
        t0 = time.perf_counter()
        u = np.random.uniform(size=n_ties)
        t1 = time.perf_counter()
        d_u = _device.to_device(u)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        del counts, d_u
        emit(score="rankhist ties", dtype=np.dtype(dt).name, n_ties=n_ties, draw_ms=round((t1 - t0) * 1e3, 3),
             upload_ms=round((t2 - t1) * 1e3, 3))
        if "--no-reference" not in sys.argv:
            ref = reference()
            if ref is None:
                emit(reference="not importable")
                continue
            ps, es = ref
            for name, fn in (("CRPS", lambda: ps.CRPS_accum(ps.CRPS_init(), X_f, X_o)),
                             ("rankhist", lambda: es.rankhist_accum(es.rankhist_init(K, 0.1), X_f, X_o)),
                             ("reldiag", lambda: ps.reldiag_accum(ps.reldiag_init(1.0), P, X_o)),
                             ("ROC", lambda: ps.ROC_curve_accum(ps.ROC_curve_init(1.0), P, X_o))):
                t0 = time.perf_counter()
                fn()
                emit(score=name, dtype=np.dtype(dt).name, reference_cpu_s=round(time.perf_counter() - t0, 3),
                     cpus=os.cpu_count())
    # CRPS above 32 members sorts in an HBM scratch plane: k = 300 at 1024^2, device-tensor input
    f = torch.rand((300, 1024, 1024), device="cuda", dtype=torch.float32)
    o = torch.rand((1024, 1024), device="cuda", dtype=torch.float32)
    fn = lambda: probscores.CRPS_accum(probscores.CRPS_init(), f, o)  # noqa: E731
    emit(score="CRPS", dtype="float32", input="tensor", members=300, size=1024, call_ms=round(wall_ms(fn), 3),
         kernels_ms=traced_ms(fn))
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "verification_timing.jsonl"), "w") as fh:
            for ln in lines:
                fh.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
