"""Time the deterministic and spatial verification scores (pysteps_b200.verification) at 2048^2, rain
with about 60 % exact zeros and 1 % NaN, float32 and float64, device-tensor input: the wall time of a
whole det_cat_fct_accum, det_cont_fct_accum (online scores, axis None and a 12-step stack over axes
(1, 2)) and fss_accum (thr 1, scale 16) call (medians of 5, synchronised) and the CUDA-event time of
each C-ABI call inside it; ensemble_spread and ensemble_skill with "fss" at 24 members, with the
kernels of one call split by name (torch.profiler: the two filter passes, the leaf sums and the
combine).  Prints one JSON line per measurement, with the card, its power limit and SM clocks read in
the same run, and also writes them to $OUT/detscores_timing.jsonl when OUT names a directory.

    python tools/detscores_timing.py              # the device (needs a GPU)
    python tools/detscores_timing.py --reference  # the reference's CPU time for the same calls, once each
"""
import json
import os
import re
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tests")]

OUT = os.environ.get("OUT")
K, SIZE, T = 24, 2048, 12
lines = []


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def fields(dt):
    from verification_cases import rain
    rng = np.random.default_rng(0)
    return (rain(rng, (K, SIZE, SIZE), dt, zeros=0.6, nans=0.01), rain(rng, (SIZE, SIZE), dt, zeros=0.6, nans=0.01),
            rain(rng, (T, SIZE, SIZE), dt, zeros=0.6, nans=0.01))


def calls(mods, E, o, S):
    """name -> the call, for the reference's modules or this package's"""
    cat, cont, spat, ens = mods
    return {
        "det_cat_fct_accum": lambda: cat.det_cat_fct_accum(cat.det_cat_fct_init(1.0), E[0], o),
        "det_cont_fct_accum": lambda: cont.det_cont_fct_accum(cont.det_cont_fct_init(), E[0], o),
        "det_cont_fct_accum T=12 axis=(1,2)": lambda: cont.det_cont_fct_accum(cont.det_cont_fct_init((1, 2)), S, E[:T]),
        "fss_accum": lambda: spat.fss_accum(spat.fss_init(1.0, 16), E[0], o),
        "ensemble_spread fss": lambda: ens.ensemble_spread(E, "fss", thr=1.0, scale=16),
        "ensemble_skill fss": lambda: ens.ensemble_skill(E, o, "fss", thr=1.0, scale=16),
    }


def reference_times():
    import importlib
    from verification_cases import reference
    if reference() is None:
        raise SystemExit("detscores_timing: the reference is not importable")
    mods = [importlib.import_module("pysteps.verification." + m)
            for m in ("detcatscores", "detcontscores", "spatialscores", "ensscores")]
    for dt in (np.float32, np.float64):
        E, o, S = fields(dt)
        for name, fn in calls(mods, E, o, S).items():
            t0 = time.perf_counter()
            fn()
            emit(call=name, dtype=np.dtype(dt).name, reference_cpu_s=round(time.perf_counter() - t0, 3),
                 cpus=os.cpu_count())


def device_times():
    import torch
    from pysteps_b200 import _device, _lib
    from pysteps_b200.verification import detcatscores, detcontscores, ensscores, spatialscores
    if not torch.cuda.is_available():
        raise SystemExit("detscores_timing: no CUDA device")
    _device.require_cuda()
    emit(card=card())

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
        """median over calls of the summed CUDA-event time of every C-ABI entry point"""
        per = {}
        for _ in range(reps):
            with _lib.Trace() as tr:
                fn()
            for name, v in tr.summary().items():
                per.setdefault(name, []).append(sum(v))
        return {name: round(statistics.median(v), 4) for name, v in per.items()}

    def kernels_ms(fn):
        """the device time of every kernel of one call, by kernel name (torch.profiler)"""
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        out = {}
        for ev in prof.key_averages():
            if ev.device_time_total > 0 and "Memcpy" not in ev.key and "Memset" not in ev.key:
                m = re.search(r"(\w+_kernel)", ev.key)
                name = m.group(1) if m else ev.key[:60]
                out[name] = round(out.get(name, 0.0) + ev.device_time_total / 1e3, 4)
        return out

    mods = (detcatscores, detcontscores, spatialscores, ensscores)
    for dt in (np.float32, np.float64):
        E, o, S = (torch.from_numpy(a).cuda() for a in fields(dt))
        for name, fn in calls(mods, E, o, S).items():
            row = dict(call=name, dtype=np.dtype(dt).name, input="tensor", size=SIZE, call_ms=round(wall_ms(fn), 3),
                       entry_points_ms=traced_ms(fn))
            if name.startswith("ensemble"):
                row.update(members=K, kernels_ms=kernels_ms(fn))
            emit(**row)
        del E, o, S
        torch.cuda.empty_cache()


def main():
    if "--reference" in sys.argv:
        reference_times()
    else:
        device_times()
    if OUT and os.path.isdir(OUT):
        with open(os.path.join(OUT, "detscores_timing.jsonl"), "w") as fh:
            for ln in lines:
                fh.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
