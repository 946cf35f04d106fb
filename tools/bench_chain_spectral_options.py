#!/usr/bin/env python
"""bench_chain_spectral_options.py -- the full-row analysis chain with one CheapTrick / D4C option per utterance.

The batch of tools/bench_spectral_options.py (synthetic 48 kHz speech, every utterance at the speaker-like Harvest
range of tools/bench_f0_ranges.py and the CheapTrick option of that range's floor: f0_floor = floor, fft_size =
GetFFTSizeForCheapTrick(fs, option); D4C at the same size), but through the whole chain with full rows out: Harvest,
CheapTrick and D4C on device arrays.  Full rows are large (at 48 kHz a 30 s utterance at fft_size 4096 takes 98 MB per
array), so the default is 128 utterances: about 25 GB for the two arrays.  The same batch is timed three ways,
alternating, with the same steps:

  mixed       world_b200_analyze_batch_spectral_options, rows of the largest size's fft_size / 2 + 1
  per_group   world_b200_analyze_batch_options once per FFT size on that size's utterances (gathered into their own
              array beforehand), rows of that size's width, their times added up
  union       world_b200_analyze_batch_options on the whole batch at the largest size

All three use the per-utterance Harvest ranges.  After the timing, the first two utterances of every size group are run
alone with the one-option chain and their rows compared with the mixed call's, bit for bit.  Device memory in use (the
whole device, as cudaMemGetInfo reports it) is recorded after each leg.  Prints ONE JSON line; writes nothing.

  python tools/bench_chain_spectral_options.py [--utts 128] [--seconds 30] [--fs 48000] [--steps 2] [--warmup 1]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=128)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--fs", type=int, default=48000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    from world_b200.api import World, HarvestOption, F0_HARVEST
    from synth import synth_batch
    from bench_f0_ranges import mixed_f0_range, gpu_info

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x = torch.empty((U, n), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 64):
        u1 = min(U, u0 + 64)
        x[u0:u1] = synth_batch(range(u0 + 1, u1 + 1), fs, n, device=dev)
    ranges = [mixed_f0_range(s) for s in range(1, U + 1)]
    ho = []
    for lo, hi in ranges:
        o = HarvestOption()
        o.f0_floor, o.f0_ceil, o.frame_period = lo, hi, 5.0
        ho.append(o)
    co = []
    for lo, _ in ranges:
        o = w.cheaptrick_option(fs)
        o.f0_floor = lo
        o.fft_size = w.lib.GetFFTSizeForCheapTrick(fs, C.byref(o))
        co.append(o)
    sizes = [o.fft_size for o in co]
    groups = {}
    for u, s in enumerate(sizes):
        groups.setdefault(s, []).append(u)
    big = max(sizes)
    W = big // 2 + 1
    ao = w.analysis_option(fs, F0_HARVEST)
    ao_union = w.analysis_option(fs, F0_HARVEST)
    ao_union.cheaptrick = co[sizes.index(big)]
    L = w.frames(fs, n, 5.0)
    t = torch.zeros((U, L), dtype=torch.float64, device=dev)
    f0 = torch.zeros((U, L), dtype=torch.float64, device=dev)
    sp = torch.zeros((U, L, W), dtype=torch.float64, device=dev)
    ap_ = torch.zeros((U, L, W), dtype=torch.float64, device=dev)
    gx = {}
    for s, idx in groups.items():
        i = torch.tensor(idx, device=dev)
        aog = w.analysis_option(fs, F0_HARVEST)
        aog.cheaptrick = co[idx[0]]
        gx[s] = (x[i].contiguous(), [ho[u] for u in idx], aog)
    free, total = torch.cuda.mem_get_info(dev)
    # the lanes' scratch: half of what is left (each lane takes half of the budget)
    w.set_scratch_budget(int(min(64 << 30, max(2 << 30, free * 0.5))))
    torch.cuda.synchronize()

    def rows(m, width):
        """[m, L, width] views at the start of the full arrays (a group's rows, packed at its own width)"""
        k = m * L * width
        return sp.view(-1)[:k].view(m, L, width), ap_.view(-1)[:k].view(m, L, width)

    def mixed():
        w.analyze_batch(x, fs, ao, time_axis=t, f0=f0, spectrogram=sp, aperiodicity=ap_, harvest_options=ho,
                        cheaptrick_options=co)

    def per_group():   # each group's rows overwrite the start of the full arrays
        for s, (xs, hs, aog) in gx.items():
            m = xs.shape[0]
            gs, ga = rows(m, s // 2 + 1)
            w.analyze_batch(xs, fs, aog, time_axis=t[:m], f0=f0[:m], spectrogram=gs, aperiodicity=ga,
                            harvest_options=hs)

    def union():
        w.analyze_batch(x, fs, ao_union, time_axis=t, f0=f0, spectrogram=sp, aperiodicity=ap_, harvest_options=ho)

    legs = {"mixed": mixed, "per_group": per_group, "union": union}
    for fn in legs.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in legs}
    in_use = {}
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
            f, tot = torch.cuda.mem_get_info(dev)
            in_use[k] = max(in_use.get(k, 0.0), (tot - f) / 1e9)
    mixed()
    w.synchronize()
    # the check: the first two utterances of each size group alone, with the one-option chain
    checked, equal = [], True
    for s, idx in sorted(groups.items()):
        sel = idx[:2]
        aog = w.analysis_option(fs, F0_HARVEST)
        aog.cheaptrick = co[sel[0]]
        tg, fg, sg, ag, _ = w.analyze_batch(x[torch.tensor(sel, device=dev)].contiguous(), fs, aog,
                                            harvest_options=[ho[u] for u in sel])
        w.synchronize()
        b = s // 2 + 1
        for j, u in enumerate(sel):
            equal = equal and all(torch.equal(p, q) for p, q in ((t[u], tg[j]), (f0[u], fg[j]), (sp[u, :, :b], sg[j]),
                                                               (ap_[u, :, :b], ag[j])))
            checked.append(u)
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    out = {"metric": "analysis frames/sec, Harvest+CheapTrick+D4C to full rows, one option per utterance",
           "value": U * L / (mean["mixed"] / 1e3), "unit": "frames/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch, per-speaker Harvest ranges, full rows "
                       f"at row_stride {W}, one GPU",
           "steps": a.steps, "warmup": a.warmup, "gpu": gpu_info(),
           "fft_sizes": {str(s): len(idx) for s, idx in sorted(groups.items())},
           "ms_per_step": ms, "mixed_over_per_group": mean["mixed"] / mean["per_group"],
           "mixed_over_union": mean["mixed"] / mean["union"],
           "device_memory_gb": {"outputs": 2 * sp.numel() * 8 / 1e9, "input": x.numel() * 8 / 1e9,
                                "device_total": total / 1e9, "in_use_after_leg": in_use},
           "check": {"rows": checked, "equal_to_one_option_chain": equal}}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
