#!/usr/bin/env python
"""bench_d4c.py -- D4C alone on one GPU, timed with CUDA events.

The batch is bench.py's config 3 by default (1024 x 10 s of synthetic 16 kHz speech); `--fs 48000 --seconds 30
--utts 256` gives the shape of config 4.  The f0 contour comes from the library's Harvest, computed once before the
timed region, so only world_b200_d4c_batch is timed.  Prints ONE JSON line: ms per call (every timed call and their
mean), the library's per-kernel CUDA-event times of the timed calls (profile_report, a separate pass so that the
per-launch events do not slow the timed one) and the card's name, power limit and SM clocks read in the same run
(read-only nvidia-smi queries).  Writes nothing.

  python tools/bench_d4c.py [--fs 16000] [--seconds 10] [--utts 1024] [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:   # the figure is informative only
        return {"error": str(e)[:100]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from world_b200.api import World
    from synth import synth_batch

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x = torch.empty((U, n), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 64):
        u1 = min(U, u0 + 64)
        x[u0:u1] = synth_batch(range(u0 + 1, u1 + 1), fs, n, device=dev)
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(min(96 << 30, max(2 << 30, free * 0.45))))
    t, f0, _ = w.harvest(x, fs)
    fft_size = w.cheaptrick_option(fs).fft_size
    ap_out = torch.empty((U, f0.shape[1], fft_size // 2 + 1), dtype=torch.float64, device=dev)
    w.trim()   # Harvest's scratch is not D4C's
    for _ in range(a.warmup):
        w.d4c(x, fs, t, f0, fft_size, out=ap_out)
    w.synchronize()
    times = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        w.d4c(x, fs, t, f0, fft_size, out=ap_out)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    w.profile(True)
    for _ in range(a.steps):
        w.d4c(x, fs, t, f0, fft_size, out=ap_out)
    w.synchronize()
    w.profile(False)
    prof = w.profile_report()
    voiced = int((f0 > 0).sum().item())
    print(json.dumps({
        "metric": "d4c_ms_per_call", "value": round(sum(times) / len(times), 3),
        "ms": [round(v, 3) for v in times],
        "shape": {"utts": U, "seconds": a.seconds, "fs": fs, "frames": U * int(f0.shape[1]), "voiced": voiced},
        "kernels": {k: {"ms_per_call": round(v["ms"] / a.steps, 3), "launches_per_call": v["launches"] / a.steps}
                    for k, v in prof.items()},
        "gpu": gpu_info(),
        "lib": os.path.basename(w.lib._name),
    }))


if __name__ == "__main__":
    main()
