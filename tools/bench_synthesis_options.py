#!/usr/bin/env python
"""bench_synthesis_options.py -- Synthesis from coded rows with one FFT size per utterance, on one GPU.

The workload of tools/bench_spectral_options.py (256 x 30 s of synthetic 48 kHz speech, each utterance with the
speaker-like F0 range of tools/bench_f0_ranges.py and the CheapTrick size of that range's floor: 4096 and 2048 at
48 kHz).  The coded rows (60 dimensions + band aperiodicities) come from world_b200_analyze_coded_batch_spectral_options
with DIO (not timed).  Output: 16-bit PCM.  Timed, alternating, with the same steps:

  mixed      world_b200_synthesis_coded_batch_options on the whole batch, one call
  per_size   world_b200_synthesis_coded_batch_modified once per size on that size's utterances (gathered into their own
             arrays beforehand), the times added up
  union      world_b200_synthesis_coded_batch_modified on the whole batch at the largest size
  union_old  the same call on the library given by --old-lib (the build of the parent change), loaded in the same
             process: the one-size path before and after, alternated in one session

The mixed rows of each size are checked against the per-size call bit for bit, and (with --old-lib) the union rows of
the two builds against each other.  Prints ONE JSON line; writes nothing.

  python tools/bench_synthesis_options.py [--utts 256] [--seconds 30] [--fs 48000] [--steps 2] [--warmup 1]
                                          [--old-lib PATH]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

DIMS = 60


def load_older(path):
    """A World on an older build of the library: only the symbols that build has are bound."""
    import world_b200.api as api
    full = api.ABI
    lib = C.CDLL(path)
    api.ABI = {k: v for k, v in full.items() if hasattr(lib, k)}
    try:
        return api.World(device=0, lib_path=path)
    finally:
        api.ABI = full


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--fs", type=int, default=48000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--old-lib", default=None, help="a second build of the library, timed on the one-size call")
    a = ap.parse_args()
    import torch
    from world_b200.api import World, DioOption, F0_DIO_STONEMASK
    from synth import synth_batch
    from bench_f0_ranges import mixed_f0_range, gpu_info

    info = gpu_info()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    old = load_older(a.old_lib) if a.old_lib else None
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    free, _ = torch.cuda.mem_get_info(dev)
    budget = int(min(64 << 30, max(2 << 30, free * 0.25)))
    for ww in (w, old):
        if ww is not None:
            ww.set_scratch_budget(budget)
    ranges = [mixed_f0_range(s) for s in range(1, U + 1)]
    co = []
    for lo, _ in ranges:
        o = w.cheaptrick_option(fs)
        o.f0_floor = lo
        o.fft_size = w.lib.GetFFTSizeForCheapTrick(fs, C.byref(o))
        co.append(o)
    sizes = [o.fft_size for o in co]
    # coded rows: DIO + StoneMask at each range, CheapTrick / D4C at each size (not timed)
    ao = w.analysis_option(fs, F0_DIO_STONEMASK)
    L = w.frames(fs, n, ao.dio.frame_period)
    n_ap = max(1, w.number_of_aperiodicities(fs))
    f0 = torch.zeros((U, L), dtype=torch.float64, device=dev)
    csp = torch.zeros((U, L, DIMS), dtype=torch.float64, device=dev)
    cap = torch.zeros((U, L, n_ap), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        x = synth_batch(range(u0 + 1, u1 + 1), fs, n, device=dev)
        do = []
        for lo, hi in ranges[u0:u1]:
            o = DioOption()
            w.lib.InitializeDioOption(C.byref(o))
            o.f0_floor, o.f0_ceil = lo, hi
            do.append(o)
        _, ff, cs, ca, _ = w.analyze_coded_batch(x, 0, fs, ao, DIMS, dio_options=do, cheaptrick_options=co[u0:u1])
        f0[u0:u1], csp[u0:u1], cap[u0:u1] = ff, cs, ca
        del x
    w.synchronize()
    groups = {}
    for u, s in enumerate(sizes):
        groups.setdefault(s, []).append(u)
    gx = {}
    for s, idx in groups.items():
        i = torch.tensor(idx, device=dev)
        gx[s] = (i, f0[i].contiguous(), csp[i].contiguous(), cap[i].contiguous())
    big = max(sizes)
    y = torch.zeros((U, n), dtype=torch.int16, device=dev)
    y_ref = torch.zeros_like(y)
    torch.cuda.synchronize()

    def mixed():
        y.copy_(w.synthesis_coded(f0, csp, cap, sizes, ao.dio.frame_period, fs, n, dtype="int16"))

    def per_size():
        for s, (i, ff, cs, ca) in gx.items():
            y_ref[i] = w.synthesis_coded(ff, cs, ca, s, ao.dio.frame_period, fs, n, dtype="int16")

    def union_with(lib):
        return lambda: lib.synthesis_coded(f0, csp, cap, big, ao.dio.frame_period, fs, n, dtype="int16")

    legs = {"mixed": mixed, "per_size": per_size, "union": union_with(w)}
    if old is not None:
        legs["union_old"] = union_with(old)
    for fn in legs.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in legs}
    for _ in range(2):   # two alternating rounds of a.steps steps per leg
        for k, fn in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / a.steps)
    mixed()
    per_size()
    torch.cuda.synchronize()
    checks = {"mixed_equals_per_size": bool(torch.equal(y, y_ref))}
    if old is not None:
        checks["union_new_equals_old"] = bool(torch.equal(legs["union"](), legs["union_old"]()))
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    out = {"metric": "synthesised samples/sec, coded rows to 16-bit PCM, one FFT size per utterance",
           "value": U * n / (mean["mixed"] / 1e3), "unit": "samples/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch, DIO f0 at per-speaker ranges and "
                       f"CheapTrick / D4C at each range's size (not timed), {DIMS} dimensions, one GPU",
           "steps": a.steps, "warmup": a.warmup, "gpu": info,
           "fft_sizes": {str(s): len(idx) for s, idx in sorted(groups.items())},
           "ms_per_step": ms, "mixed_over_per_size": mean["mixed"] / mean["per_size"],
           "mixed_over_union": mean["mixed"] / mean["union"],
           "union_over_union_old": mean["union"] / mean["union_old"] if old is not None else None,
           "checks": checks}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
