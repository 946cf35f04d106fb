#!/usr/bin/env python
"""bench_harvest_sweep.py -- Harvest alone on one GPU, timed with CUDA events.

The batch is bench.py's config 3 by default (1024 x 10 s of synthetic 16 kHz speech); `--ranges mixed` gives every
utterance the per-utterance F0 range that tools/bench_f0_ranges.py picks for it (one world_b200_harvest_batch_options
call).  Only the Harvest call is timed.  Prints ONE JSON line: ms per call (every timed call and their mean), the
library's per-kernel CUDA-event times of the timed calls (profile_report, a separate pass so that the per-launch
events do not slow the timed one) with the band sweep's two kernels, band_fir_events_kernel and band_interp_kernel,
pulled out, and the card's name, power limit and SM clocks read in the same run (read-only nvidia-smi queries).
Writes nothing unless `--dump DIR` is given: then the time axis and f0 of the last call go to DIR as float64 .npy,
so that two builds can be compared value for value on the same batch.

  python tools/bench_harvest_sweep.py [--fs 16000] [--seconds 10] [--utts 1024] [--ranges default|mixed]
                                      [--steps 5] [--warmup 2] [--dump DIR]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SWEEP_KERNELS = ("band_fir_events_kernel", "band_interp_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--ranges", default="default", choices=["default", "mixed"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dump", metavar="DIR", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from world_b200.api import World, HarvestOption
    from synth import synth_batch
    from bench_d4c import gpu_info
    from bench_f0_ranges import mixed_f0_range

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x = torch.empty((U, n), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 64):
        u1 = min(U, u0 + 64)
        x[u0:u1] = synth_batch(range(u0 + 1, u1 + 1), fs, n, device=dev)
    option = None
    if a.ranges == "mixed":
        option = []
        for s in range(1, U + 1):
            o = HarvestOption()
            o.f0_floor, o.f0_ceil = mixed_f0_range(s)
            o.frame_period = w.harvest_option().frame_period
            option.append(o)
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(min(96 << 30, max(2 << 30, free * 0.45))))
    for _ in range(a.warmup):
        w.harvest(x, fs, option)
    w.synchronize()
    times = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        t, f0, _ = w.harvest(x, fs, option)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    w.profile(True)
    for _ in range(a.steps):
        w.harvest(x, fs, option)
    w.synchronize()
    w.profile(False)
    prof = w.profile_report()
    kernels = {k: {"ms_per_call": round(v["ms"] / a.steps, 3), "launches_per_call": v["launches"] / a.steps}
               for k, v in prof.items()}
    if a.dump:
        os.makedirs(a.dump, exist_ok=True)
        np.save(os.path.join(a.dump, "time_axis.npy"), t.cpu().numpy())
        np.save(os.path.join(a.dump, "f0.npy"), f0.cpu().numpy())
    print(json.dumps({
        "metric": "harvest_ms_per_call", "value": round(sum(times) / len(times), 3),
        "ms": [round(v, 3) for v in times],
        "sweep": {k: kernels.get(k, {}).get("ms_per_call") for k in SWEEP_KERNELS},
        "shape": {"utts": U, "seconds": a.seconds, "fs": fs, "ranges": a.ranges, "frames": U * int(f0.shape[1]),
                  "voiced": int((f0 > 0).sum().item())},
        "kernels": kernels,
        "gpu": gpu_info(),
        "lib": os.path.basename(w.lib._name),
    }))


if __name__ == "__main__":
    main()
