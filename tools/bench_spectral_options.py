#!/usr/bin/env python
"""bench_spectral_options.py -- one CheapTrick / D4C option (so one FFT size) per utterance on one GPU.

The shape of bench.py's config 4 (256 x 30 s of synthetic 48 kHz speech, CheapTrick + D4C on a precomputed f0), with
coded rows out (60 dimensions + band aperiodicities).  Every utterance gets the speaker-like Harvest range of
tools/bench_f0_ranges.py (its f0 comes from Harvest at that range, not timed) and the CheapTrick option of that range's
floor: f0_floor = floor, fft_size = GetFFTSizeForCheapTrick(fs, option); D4C runs at the same size.  The same batch is
timed three ways, alternating, with the same steps:

  mixed       world_b200_cheaptrick_coded_batch_options + world_b200_d4c_coded_batch_options, one call each
  per_group   world_b200_cheaptrick_coded_batch + world_b200_d4c_coded_batch once per FFT size on that size's
              utterances (gathered into their own array beforehand), their times added up
  union       world_b200_cheaptrick_coded_batch + world_b200_d4c_coded_batch on the whole batch at the largest size

and rows of the mixed result are checked against the reference's CheapTrick / D4C at each row's own option, coded by
the reference's CodeSpectralEnvelope / CodeAperiodicity.  Prints ONE JSON line; writes nothing.

  python tools/bench_spectral_options.py [--utts 256] [--seconds 30] [--fs 48000] [--steps 3] [--warmup 1]
                                         [--no-parity]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--fs", type=int, default=48000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-parity", action="store_true",
                    help="skip the check of row 0 and the first row of every size group against the reference")
    a = ap.parse_args()
    import numpy as np
    import torch
    from world_b200.api import World, HarvestOption
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
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(min(96 << 30, max(2 << 30, free * 0.3))))
    # the f0 rows: Harvest at each utterance's range (not timed)
    L = w.frames(fs, n, 5.0)
    t = torch.empty((U, L), dtype=torch.float64, device=dev)
    f0 = torch.empty((U, L), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        ho = []
        for lo, hi in ranges[u0:u1]:
            o = HarvestOption()
            o.f0_floor, o.f0_ceil, o.frame_period = lo, hi, 5.0
            ho.append(o)
        tt, ff, _ = w.harvest(x[u0:u1], fs, ho)
        t[u0:u1], f0[u0:u1] = tt, ff
    w.synchronize()

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
    gx = {}
    for s, idx in groups.items():
        i = torch.tensor(idx, device=dev)
        gx[s] = (x[i].contiguous(), t[i].contiguous(), f0[i].contiguous(), co[idx[0]])
    big = max(sizes)
    co_union = co[sizes.index(big)]
    n_ap = max(1, w.number_of_aperiodicities(fs))
    csp = torch.zeros((U, L, DIMS), dtype=torch.float64, device=dev)
    cap = torch.zeros((U, L, n_ap), dtype=torch.float64, device=dev)
    torch.cuda.synchronize()

    def mixed():
        csp.copy_(w.cheaptrick_coded(x, fs, t, f0, DIMS, co))
        cap.copy_(w.d4c_coded(x, fs, t, f0, sizes))

    def per_group():   # outputs in group order: rows [off, off + m) hold group s
        off = 0
        for s, (xs, ts, fs_, o) in gx.items():
            m = xs.shape[0]
            csp[off:off + m] = w.cheaptrick_coded(xs, fs, ts, fs_, DIMS, o)
            cap[off:off + m] = w.d4c_coded(xs, fs, ts, fs_, s)
            off += m

    def union_call():
        csp.copy_(w.cheaptrick_coded(x, fs, t, f0, DIMS, co_union))
        cap.copy_(w.d4c_coded(x, fs, t, f0, big))

    legs = {"mixed": mixed, "per_group": per_group, "union": union_call}
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
    w.synchronize()
    parity = None
    if not a.no_parity:
        from refworld import RefWorld, REF_LIB, ORACLE_LIB, rel_err
        ref = RefWorld(REF_LIB if os.path.exists(REF_LIB) else ORACLE_LIB)
        rows = sorted({0} | {idx[0] for idx in groups.values()})
        worst = {"coded_sp": 0.0, "coded_ap": 0.0}
        for r in rows:
            xu = np.ascontiguousarray(x[r].cpu().numpy())
            tu, fu = t[r].cpu().numpy(), f0[r].cpu().numpy()
            ro = ref.cheaptrick_option(fs)
            ro.f0_floor, ro.fft_size = ranges[r][0], sizes[r]
            want_sp = ref.code_spectral_envelope(ref.cheaptrick(xu, fs, tu, fu, ro), fs, sizes[r], DIMS)
            want_ap = ref.code_aperiodicity(ref.d4c(xu, fs, tu, fu, sizes[r]), fs, sizes[r])
            for name, got, want in (("coded_sp", csp[r], want_sp), ("coded_ap", cap[r], want_ap)):
                want = np.asarray(want)
                e = rel_err(got.cpu().numpy(), want, floor=1e-4 * np.abs(want).max()).max()
                worst[name] = max(worst[name], float(e))
        parity = {"against": f"{os.path.basename(ref.lib._name)} CheapTrick / D4C at each row's own option, "
                             "coded by its CodeSpectralEnvelope / CodeAperiodicity",
                  "rows": rows, "max_rel_err": worst,
                  "tolerance": "1e-6 relative, floored at 1e-4 of the row's largest magnitude",
                  "within_tolerance": max(worst.values()) <= 1e-6}
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    out = {"metric": "analysis frames/sec, CheapTrick+D4C to coded rows, one option per utterance",
           "value": U * L / (mean["mixed"] / 1e3), "unit": "frames/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch, f0 from Harvest at per-speaker ranges "
                       f"(not timed), {DIMS} dimensions, one GPU",
           "steps": a.steps, "warmup": a.warmup, "gpu": gpu_info(),
           "fft_sizes": {str(s): len(idx) for s, idx in sorted(groups.items())},
           "ms_per_step": ms, "mixed_over_per_group": mean["mixed"] / mean["per_group"],
           "mixed_over_union": mean["mixed"] / mean["union"], "parity": parity}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
