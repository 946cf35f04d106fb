#!/usr/bin/env python
"""bench_packed_synthesis.py -- the way back on packed rows against the padded calls, on a corpus of mixed lengths.

The corpus of tools/bench_packed.py (N utterances of synthetic speech, lengths log-uniform in [1, 30] s, the same seed).
Features are made once: coded rows (60 dimensions) with analyze_coded_packed and full rows with analyze_packed, Harvest
-> CheapTrick (fft_size 1024 at 16 kHz) -> D4C, then scattered into padded [n][L][...] rows for the padded legs.  Three
pairs of calls, timed alternating in one session:

  coded    synthesis_coded_packed int16 (f0 [F], coded rows [F][dims])  vs  synthesis_coded (options) int16 on padded rows
  full     synthesis_packed (full rows [F][bins])                       vs  synthesis (options) on padded rows
  host     synthesis_coded_host_packed  vs  synthesis_coded_host (options), HOST arrays, int16 into pinned buffers

Reports per leg: ms per call in each round (CUDA events around `steps` calls), passes per call (syn_timebase_kernel
launches, from world_b200_profile_report in a run of its own), device memory in use (cudaMemGetInfo) after the leg's
timed rounds and after one call made with the library's buffers given back first, the
bytes the host legs move over PCIe (counted from the shapes each call copies), a bit-equality check of the first
utterances, and the card's name, power limit and SM clock during the timing.  Prints ONE JSON line; writes nothing.

  python tools/bench_packed_synthesis.py [--utts 512] [--fs 16000] [--steps 1] [--warmup 1] [--rounds 3]
                                         [--scratch-gb 8]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

DIMS = 60


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=512)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--check", type=int, default=8, help="utterances compared bit for bit")
    ap.add_argument("--scratch-gb", type=float, default=8.0, help="the library's scratch budget for the legs")
    a = ap.parse_args()

    import torch
    from world_b200.api import World, F0_HARVEST
    from synth import synth_batch
    from bench import ClockSampler
    from bench_f0_ranges import gpu_info
    from bench_packed import corpus_lengths

    if not torch.cuda.is_available():
        raise SystemExit("bench_packed_synthesis.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, U = a.fs, a.utts
    lens = corpus_lengths(U, fs)
    S, M = sum(lens), max(lens)
    xo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x = torch.empty(S, dtype=torch.float64, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        xb = synth_batch(range(u0 + 1, u1 + 1), fs, max(lens[u0:u1]), device=dev)
        for u in range(u0, u1):
            x[xo[u]:xo[u + 1]] = xb[u - u0, :lens[u]]
    del xb
    ao = w.analysis_option(fs, F0_HARVEST)
    fft, fp = ao.cheaptrick.fft_size, ao.harvest.frame_period
    bins = fft // 2 + 1
    _, f0, csp, cap, fo = w.analyze_coded_packed(x, 0, xo, fs, ao, DIMS)
    _, _, sp, apr, _ = w.analyze_packed(x, xo, fs, ao)
    w.synchronize()
    del x
    F = int(fo[-1])
    fl = [int(v) for v in np.diff(fo)]
    L = max(fl)
    n_ap = w.number_of_aperiodicities(fs)
    sizes = [fft] * U

    def pad(a):   # packed [F, ...] -> padded [U, L, ...]
        out = torch.zeros((U, L) + tuple(a.shape[1:]), dtype=a.dtype, device=a.device)
        for u in range(U):
            out[u, :fl[u]] = a[fo[u]:fo[u + 1]]
        return out

    # the analysis arenas go back; every leg then works within the same scratch budget, next to both layouts' inputs
    w.trim()
    w.set_scratch_budget(int(a.scratch_gb * (1 << 30)))
    pf0, pcsp, pcap = pad(f0), pad(csp), pad(cap)
    psp, pap = pad(sp), pad(apr)
    hf0, hcsp, hcap = f0.cpu().numpy(), csp.cpu().numpy(), cap.cpu().numpy()
    hpf0, hpcsp, hpcap = pf0.cpu().numpy(), pcsp.cpu().numpy(), pcap.cpu().numpy()
    y_host_packed = torch.empty(S, dtype=torch.int16).pin_memory().numpy()
    y_host_padded = torch.empty((U, M), dtype=torch.int16).pin_memory().numpy()
    outs = {}

    legs = {
        "coded_packed": lambda: outs.__setitem__("coded_packed", w.synthesis_coded_packed(
            f0, csp, cap, fo, sizes, fp, fs, xo, dtype="int16")),
        "coded_padded": lambda: outs.__setitem__("coded_padded", w.synthesis_coded(
            pf0, pcsp, pcap, sizes, fp, fs, M, f0_lengths=fl, y_lengths=lens, dtype="int16")),
        "full_packed": lambda: outs.__setitem__("full_packed", w.synthesis_packed(
            f0, sp, apr, fo, sizes, fp, fs, xo)),
        "full_padded": lambda: outs.__setitem__("full_padded", w.synthesis(
            pf0, psp, pap, sizes, fp, fs, M, f0_lengths=fl, y_lengths=lens)),
        "host_packed": lambda: w.synthesis_coded_host_packed(hf0, hcsp, hcap, fo, sizes, fp, fs, xo, nbit=16,
                                                             out=y_host_packed),
        "host_padded": lambda: w.synthesis_coded_host(hpf0, hpcsp, hpcap, sizes, fp, fs, M, nbit=16, f0_lengths=fl,
                                                      y_lengths=lens, out=y_host_padded),
    }
    for fn in legs.values():
        for _ in range(a.warmup):
            fn()
            w.synchronize()
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    sampler.start()
    ms = {k: [] for k in legs}
    in_use = {}
    for _ in range(a.rounds):
        for k, fn in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / a.steps)
            free, total = torch.cuda.mem_get_info(dev)
            in_use[k] = max(in_use.get(k, 0.0), (total - free) / 1e9)
    clocks = sampler.stop()
    # one more call of each leg on its own: the library's buffers given back first, so that the memory in use after it
    # is the inputs plus what that call needed; and its profile, whose time-base launches are its passes
    passes, own = {}, {}
    for k, fn in legs.items():
        w.trim()
        torch.cuda.empty_cache()
        w.profile(True)
        fn()
        w.synchronize()
        rep = w.profile_report()
        w.profile(False)
        free, total = torch.cuda.mem_get_info(dev)
        own[k] = (total - free) / 1e9
        passes[k] = sum(v["launches"] for n, v in rep.items() if n.startswith("syn_timebase_kernel"))
    # the first utterances of each pair, bit for bit
    for k in ("coded_packed", "coded_padded", "full_packed", "full_padded", "host_packed", "host_padded"):
        legs[k]()
    w.synchronize()
    yc, ycp = outs["coded_packed"].cpu().numpy(), outs["coded_padded"].cpu().numpy()
    yf, yfp = outs["full_packed"].cpu().numpy(), outs["full_padded"].cpu().numpy()
    equal = {"coded": True, "full": True, "host": True}
    for u in range(min(a.check, U)):
        s0, s1 = int(xo[u]), int(xo[u + 1])
        equal["coded"] &= bool(np.array_equal(yc[s0:s1], ycp[u, :lens[u]]))
        equal["full"] &= bool(np.array_equal(yf[s0:s1], yfp[u, :lens[u]]))
        equal["host"] &= bool(np.array_equal(y_host_packed[s0:s1], y_host_padded[u, :lens[u]]))
        equal["host"] &= bool(np.array_equal(y_host_packed[s0:s1], yc[s0:s1]))
    pcie = {"host_packed": {"h2d": F * (1 + DIMS + n_ap) * 8, "d2h": S * 2},
            "host_padded": {"h2d": U * L * (1 + DIMS + n_ap) * 8, "d2h": U * M * 2}}
    med = {k: statistics.median(v) for k, v in ms.items()}
    out = {"metric": "synthesis output samples/sec, packed rows vs padded rows, corpus of log-uniform 1-30 s",
           "value": S / (med["coded_packed"] / 1e3), "unit": "samples/s",
           "workload": f"{U} utterances, {fs // 1000} kHz synthetic speech, lengths log-uniform in [1, 30] s "
                       f"({S / fs:.0f} s in all), Harvest features, fft {fft}, {DIMS} coded dimensions",
           "frames_packed": F, "frames_padded": U * L, "samples_packed": S, "samples_padded": U * M,
           "ms_per_call_rounds": ms, "ms_per_call_median": med,
           "spread_pct": {k: 100.0 * (max(v) - min(v)) / statistics.median(v) for k, v in ms.items()},
           "passes_per_call": passes, "device_memory_in_use_gb_after_leg": in_use,
           "device_memory_in_use_gb_after_one_call_from_trimmed": own,
           "pcie_bytes_counted": pcie, "scratch_budget_gb": a.scratch_gb, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
           "check": {"utterances": min(a.check, U), "packed_equals_padded": equal},
           "gpu": gpu_info(), "clocks_during_timing": clocks}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
