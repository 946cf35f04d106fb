#!/usr/bin/env python
"""bench_f0_ranges.py -- one F0 range per utterance on one GPU, Harvest or DIO.

The workload of bench.py's config 3 (1024 x 10 s of synthetic 16 kHz speech, Harvest -> CheapTrick -> D4C through
the device-resident chain) or, with --f0 dio, of its config 2 (the same batch, DIO -> StoneMask -> CheapTrick -> D4C;
the other DIO settings are the defaults), with every utterance analysed at a speaker-like range of its own: the
narrowest of
MIXED_F0_RANGES (fewest channels, ties to the first listed) that holds its generated contour -- tests/synth.py gives
utterance `seed` the contour base x (1 +- 0.25), base ~ U(90, 250) Hz from the RandomState below, so the choice is
fixed by the seed.  The same batch is timed three ways, alternating, with the same steps:

  mixed       one world_b200_analyze_batch_options (--f0 dio: world_b200_analyze_batch_dio_options) call with one
              option per utterance
  per_group   one world_b200_analyze_batch call per range group, their times added up
  union       one world_b200_analyze_batch call at the union of the ranges

and rows of the mixed result are checked against the reference's own chain (its Harvest, or its Dio + StoneMask, at
the utterance's range feeding its CheapTrick and D4C).  Prints ONE JSON line; writes nothing.

  python tools/bench_f0_ranges.py [--f0 harvest|dio] [--utts 1024] [--seconds 10] [--steps 3] [--warmup 2]
                                  [--no-parity]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

MIXED_F0_RANGES = [(50.0, 300.0), (60.0, 400.0), (100.0, 600.0), (71.0, 800.0), (40.0, 1100.0)]


def harvest_channels(lo, hi):
    return 1 + int(math.log(hi * 1.1 / (lo * 0.9)) / math.log(2.0) * 40)


def dio_channels(lo, hi, channels_in_octave=2.0):
    return 1 + int(math.log(hi / lo) / math.log(2.0) * channels_in_octave)


def mixed_f0_range(seed):
    import numpy as np
    base = np.random.RandomState((1000003 * int(seed) + 17) % (1 << 32)).uniform(90.0, 250.0)
    fits = [r for r in MIXED_F0_RANGES if r[0] <= 0.75 * base and 1.25 * base <= r[1]]
    return min(fits, key=lambda r: harvest_channels(*r))


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:   # the figure is informative only
        return {"error": str(e)[:100]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--f0", default="harvest", choices=["harvest", "dio"])
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-parity", action="store_true",
                    help="skip the check of rows 0, U/2, U-1 and the first row of every range group against the reference")
    a = ap.parse_args()
    import numpy as np
    import torch
    from world_b200.api import World, DioOption, HarvestOption, F0_DIO_STONEMASK, F0_HARVEST
    from synth import synth_batch
    from bench import parity_entry, parity_summary

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x = torch.empty((U, n), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 64):
        u1 = min(U, u0 + 64)
        x[u0:u1] = synth_batch(range(u0 + 1, u1 + 1), fs, n, device=dev)
    ranges = [mixed_f0_range(s) for s in range(1, U + 1)]
    dio = a.f0 == "dio"
    method = F0_DIO_STONEMASK if dio else F0_HARVEST
    ao = w.analysis_option(fs, method)
    opts = []
    for lo, hi in ranges:
        if dio:   # the default option with the utterance's range
            o = DioOption()
            for name, _ in DioOption._fields_:
                setattr(o, name, getattr(ao.dio, name))
            o.f0_floor, o.f0_ceil = lo, hi
        else:
            o = HarvestOption()
            o.f0_floor, o.f0_ceil, o.frame_period = lo, hi, ao.harvest.frame_period
        opts.append(o)
    channels = (lambda lo, hi: dio_channels(lo, hi, ao.dio.channels_in_octave)) if dio else harvest_channels
    groups = {}
    for u, r in enumerate(ranges):
        groups.setdefault(r, []).append(u)
    union = (min(r[0] for r in groups), max(r[1] for r in groups))
    xg = {r: x[torch.tensor(idx, device=dev)].contiguous() for r, idx in groups.items()}
    L = w.frames(fs, n, ao.dio.frame_period if dio else ao.harvest.frame_period)
    bins = ao.cheaptrick.fft_size // 2 + 1
    t = torch.zeros((U, L), dtype=torch.float64, device=dev)
    f0 = torch.zeros((U, L), dtype=torch.float64, device=dev)
    sp = torch.zeros((U, L, bins), dtype=torch.float64, device=dev)
    ap_ = torch.zeros((U, L, bins), dtype=torch.float64, device=dev)
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(min(96 << 30, max(2 << 30, free * 0.45))))

    def option_for(r):
        o = w.analysis_option(fs, method)
        if dio:
            o.dio.f0_floor, o.dio.f0_ceil = r
        else:
            o.harvest.f0_floor, o.harvest.f0_ceil = r
        return o

    per_utt = {"dio_options": opts} if dio else {"harvest_options": opts}

    def mixed():
        w.analyze_batch(x, fs, ao, time_axis=t, f0=f0, spectrogram=sp, aperiodicity=ap_, **per_utt)

    def per_group():   # outputs in group order: rows [off, off + m) hold group r
        off = 0
        for r, idx in groups.items():
            m = len(idx)
            w.analyze_batch(xg[r], fs, option_for(r), time_axis=t[off:off + m], f0=f0[off:off + m],
                            spectrogram=sp[off:off + m], aperiodicity=ap_[off:off + m])
            off += m

    def union_call():
        w.analyze_batch(x, fs, option_for(union), time_axis=t, f0=f0, spectrogram=sp, aperiodicity=ap_)

    legs = {"mixed_single_call": mixed, "per_group_calls": per_group, "union_range_call": union_call}
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
    # the mixed result, for the parity check
    mixed()
    w.synchronize()
    parity = None
    rows = sorted({0, U // 2, U - 1} | {idx[0] for idx in groups.values()})
    if not a.no_parity:
        from refworld import RefWorld, REF_LIB, ORACLE_LIB
        ref = RefWorld(REF_LIB if os.path.exists(REF_LIB) else ORACLE_LIB)
        entries = []
        for r in rows:
            xu = np.ascontiguousarray(x[r].cpu().numpy())
            if dio:
                do = ref.dio_option()
                do.f0_floor, do.f0_ceil = ranges[r]
                tr, fr = ref.dio(xu, fs, do)
                fr = ref.stonemask(xu, fs, tr, fr)
            else:
                ho = ref.harvest_option()
                ho.f0_floor, ho.f0_ceil = ranges[r]
                tr, fr = ref.harvest(xu, fs, ho)
            co = ref.cheaptrick_option(fs)
            want = (tr, fr, ref.cheaptrick(xu, fs, tr, fr, co), ref.d4c(xu, fs, tr, fr, co.fft_size))
            got = (t[r].cpu().numpy(), f0[r].cpu().numpy(), sp[r].cpu().numpy(), ap_[r].cpu().numpy())
            entries.append(parity_entry(np, got, want))
        parity = parity_summary(entries, rows, "the reference's own chain at each row's own F0 range "
                                              f"({os.path.basename(ref.lib._name)})")
    frames = U * L
    chain = "Dio+StoneMask+CheapTrick+D4C" if dio else "Harvest+CheapTrick+D4C"
    out = {"metric": f"analysis frames/sec, {chain}, one F0 range per utterance",
           "value": frames / (sum(ms["mixed_single_call"]) / len(ms["mixed_single_call"]) / 1e3), "unit": "frames/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch, one GPU", "steps": a.steps,
           "warmup": a.warmup, "gpu": gpu_info(),
           "ranges": {f"{lo:g}-{hi:g} Hz": len(idx) for (lo, hi), idx in groups.items()},
           "channels": {f"{lo:g}-{hi:g} Hz": channels(lo, hi) for (lo, hi) in list(groups) + [union]},
           "union_range": f"{union[0]:g}-{union[1]:g} Hz",
           "ms_per_step": ms,
           "parity": parity}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
