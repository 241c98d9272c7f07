"""Time the constant advection method at 512^2, 2048^2 and 4096^2 (two seeded rain frames shifted by
(3, -2) px): one objective evaluation on the device (CUDA events around b200_constant_eval), a whole
motion.get_method("constant") call (host clock, NumPy input and device-tensor input), and the
reference's CPU time on the same machine -- one evaluation of its objective, and a whole call up to
2048^2.  Prints one JSON line per measurement, with the card, its power limit and SM clocks, and
also writes them to $OUT/constant_timing.jsonl when OUT names a directory.

    python tools/constant_timing.py
"""
import json
import os
import statistics
import subprocess
import sys
import time
import warnings
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "golden")]
from pysteps_b200 import _device, _lib  # noqa: E402
from pysteps_b200 import _synthetic as syn  # noqa: E402
from pysteps_b200.motion import get_method  # noqa: E402

OUT = os.environ.get("OUT")
lines = []


def emit(**kw):
    print(json.dumps(kw), flush=True)
    lines.append(kw)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def device_eval_ms(R, reps=50):
    prev, nxt = _device.to_device(R[-2]), _device.to_device(R[-1])
    m, n = prev.shape
    nbytes = _lib.c_i64(0)
    _lib.call("b200_constant_scratch_bytes", m, n, nbytes)
    scratch = torch.zeros(int(nbytes.value), dtype=torch.uint8, device="cuda")
    record = torch.empty(3, dtype=torch.float64, device="cuda")

    def once(v):
        _lib.call("b200_constant_eval", prev.data_ptr(), nxt.data_ptr(), _device.dtype_code(prev.dtype), m, n,
                  v[0], v[1], scratch.data_ptr(), record.data_ptr(), _device.stream_ptr())

    pts = [(-2.5, 1.5), (-3.0, 2.0), (0.5, 0.5)]
    for p in pts:
        once(p)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for k in range(reps):
        once(pts[k % 3])
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def wall(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out), min(out), max(out)


def reference_module():
    try:
        import _refimport
        return _refimport.ref_module("pysteps.motion.constant") if _refimport.available() else None
    except Exception:  # noqa: BLE001 -- no reference on this machine
        return None


def reference_eval_ms(ref, R, reps=3):
    """one evaluation of the reference's objective: the f handed to op.minimize, called at one point"""
    times = []

    def grab(fun, x0, **kw):
        fun(np.array([-2.5, 1.5]))
        for _ in range(reps):
            t0 = time.perf_counter()
            fun(np.array([-2.5, 1.5]))
            times.append((time.perf_counter() - t0) * 1e3)
        raise StopIteration

    with mock.patch.object(ref.op, "minimize", grab):
        try:
            ref.constant(R)
        except StopIteration:
            pass
    return statistics.median(times)


def main():
    _device.require_cuda()
    emit(card=card(), torch=torch.__version__)
    ref = reference_module()
    constant = get_method("constant")
    warnings.simplefilter("ignore")
    for size in (512, 2048, 4096):
        R = syn.rain_frames(size, size, 2, seed=1, dx=3, dy=-2)
        Rd = torch.from_numpy(R).cuda()
        constant(R)  # warm-up (allocator, first launches)
        emit(size=size, what="one evaluation, device (CUDA events, 50 calls)", ms=round(device_eval_ms(R), 4))
        med, lo, hi = wall(lambda: constant(R), 5)
        emit(size=size, what="whole call, NumPy input (host clock, 5 calls)", ms_median=round(med, 3),
             ms_min=round(lo, 3), ms_max=round(hi, 3))
        med, lo, hi = wall(lambda: constant(Rd), 5)
        emit(size=size, what="whole call, device tensor input (host clock, 5 calls)", ms_median=round(med, 3),
             ms_min=round(lo, 3), ms_max=round(hi, 3))
        if ref is not None:
            emit(size=size, what="reference: one evaluation (CPU, median of 3)", ms=round(reference_eval_ms(ref, R), 3))
            if size <= 2048:
                t0 = time.perf_counter()
                ref.constant(R)
                emit(size=size, what="reference: whole call (CPU, 1 call)", ms=round((time.perf_counter() - t0) * 1e3, 1))
    emit(card_after=card())
    if OUT:
        os.makedirs(OUT, exist_ok=True)
        with open(os.path.join(OUT, "constant_timing.jsonl"), "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
