#!/usr/bin/env python
"""bench_packed_stages.py -- the packed stage calls against the padded _options calls on a corpus of mixed lengths.

The corpus of tools/bench_packed.py: N seeded utterances of synthetic speech (tests/synth.py) whose lengths are drawn
log-uniformly from [1, 30] s.  Their F0 comes from world_b200_analyze_packed with NULL rows (Harvest, F0 stage only).
Two pairs of calls on the same utterances and F0, each pair timed alternating, three rounds:

  full     world_b200_cheaptrick_packed + world_b200_d4c_packed (x [X], time axis / f0 [F], rows [F][bins])
           vs  world_b200_cheaptrick_batch_options + world_b200_d4c_batch_options (x [n][longest], time axis / f0
           [n][L], rows [n][L][bins], L the longest utterance's frame count)
  coded    world_b200_cheaptrick_coded_packed + world_b200_d4c_coded_packed  vs  the padded *_coded_batch_options

Reports ms per call pair; each leg's device memory (cudaMemGetInfo) before and after one call from a trimmed context,
whose difference is the scratch the leg grows to, its high-water above the resident arrays (every array of both
layouts stays allocated throughout); and the counted bytes of each layout's arrays: the
padded ones are what a caller holding a packed corpus has to build to use the padded calls.  The card's name and power
limit are read in the same run; the first utterances of each pair are compared bit for bit.  Prints ONE JSON line;
writes nothing.  --count-only gives the byte counts without a GPU.

  python tools/bench_packed_stages.py [--utts 512] [--fs 16000] [--steps 1] [--warmup 1] [--dims 40] [--count-only]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_packed import corpus_lengths, frames  # noqa: E402


def counts(lens, fs, bins, dims, n_ap):
    """Bytes of the arrays each layout's calls take and give: samples, time axis and f0, full and coded rows."""
    n, fl = len(lens), [frames(fs, v) for v in lens]
    L, F, S = max(fl), sum(fl), sum(lens)
    per_frame_full = (2 + 2 * bins) * 8
    per_frame_coded = (2 + dims + n_ap) * 8
    return {"frames_padded": n * L, "frames_packed": F,
            "full_bytes": {"padded": n * max(lens) * 8 + n * L * per_frame_full, "packed": S * 8 + F * per_frame_full},
            "coded_bytes": {"padded": n * max(lens) * 8 + n * L * per_frame_coded,
                            "packed": S * 8 + F * per_frame_coded},
            "padded_over_packed_full": (n * max(lens) * 8 + n * L * per_frame_full) / (S * 8 + F * per_frame_full)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=512)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dims", type=int, default=40)
    ap.add_argument("--count-only", action="store_true")
    a = ap.parse_args()
    fs, U = a.fs, a.utts
    lens = corpus_lengths(U, fs)
    n_ap = max(0, int(min(15000.0, fs / 2.0 - 3000.0) / 3000.0))
    fft = 1 << int(np.ceil(np.log2(3.0 * fs / 71.0 + 1)))   # GetFFTSizeForCheapTrick at the default floor
    bins = fft // 2 + 1
    out = {"metric": "ms per CheapTrick + D4C call pair, packed stage calls vs padded _options calls",
           "workload": f"{U} utterances, {fs // 1000} kHz synthetic speech, lengths log-uniform in [1, 30] s, "
                       "F0 from analyze_packed (Harvest)",
           "counted": counts(lens, fs, bins, a.dims, n_ap)}
    if a.count_only:
        print(json.dumps(out), flush=True)
        return
    import torch
    from world_b200.api import World, F0_HARVEST
    from synth import synth_batch
    from bench_f0_ranges import gpu_info

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    S, M = sum(lens), max(lens)
    xo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x_packed = torch.empty(S, dtype=torch.float64, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        xb = synth_batch(range(u0 + 1, u1 + 1), fs, max(lens[u0:u1]), device=dev)
        for u in range(u0, u1):
            x_packed[xo[u]:xo[u + 1]] = xb[u - u0, :lens[u]]
    ao = w.analysis_option(fs, F0_HARVEST)
    assert ao.cheaptrick.fft_size == fft
    fo = w.packed_frames(fs, xo, 5.0)
    F, fl = int(fo[-1]), np.diff(fo)
    L = int(fl.max())
    # F0 alone: analyze_packed with NULL rows stops after the F0 stage
    t = torch.zeros(F, dtype=torch.float64, device=dev)
    f0 = torch.zeros(F, dtype=torch.float64, device=dev)
    w._use_current_stream()
    n_c, xo_c = U, (C.c_longlong * (U + 1))(*[int(v) for v in xo])
    w._check(w.lib.world_b200_analyze_packed(w._h, x_packed.data_ptr(), n_c, xo_c, fs, C.byref(ao), None, None, None,
                                             None, t.data_ptr(), f0.data_ptr(), 0, None, None, None))
    # the padded rows a caller would build from the packed corpus
    x_pad = torch.zeros((U, M), dtype=torch.float64, device=dev)
    t_pad = torch.zeros((U, L), dtype=torch.float64, device=dev)
    f0_pad = torch.zeros((U, L), dtype=torch.float64, device=dev)
    for u in range(U):
        x_pad[u, :lens[u]] = x_packed[xo[u]:xo[u + 1]]
        t_pad[u, :fl[u]] = t[fo[u]:fo[u + 1]]
        f0_pad[u, :fl[u]] = f0[fo[u]:fo[u + 1]]
    cto, d4o, sizes = [ao.cheaptrick] * U, [ao.d4c] * U, [fft] * U
    pk = [torch.zeros((F, bins), dtype=torch.float64, device=dev) for _ in range(2)]
    pd = [torch.zeros((U, L, bins), dtype=torch.float64, device=dev) for _ in range(2)]
    pkc = [torch.zeros((F, a.dims), dtype=torch.float64, device=dev),
           torch.zeros((F, max(1, n_ap)), dtype=torch.float64, device=dev)]
    pdc = [torch.zeros((U, L, a.dims), dtype=torch.float64, device=dev),
           torch.zeros((U, L, max(1, n_ap)), dtype=torch.float64, device=dev)]
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(max(2 << 30, free * 0.3)))

    def full_packed():
        w.cheaptrick_packed(x_packed, xo, fs, t, f0, fo, cto, out=pk[0])
        w.d4c_packed(x_packed, xo, fs, t, f0, fo, sizes, d4o, out=pk[1])

    def full_padded():
        w.cheaptrick(x_pad, fs, t_pad, f0_pad, cto, x_lengths=lens, f0_lengths=fl, out=pd[0])
        w.d4c(x_pad, fs, t_pad, f0_pad, sizes, d4o, x_lengths=lens, f0_lengths=fl, out=pd[1])

    def coded_packed():
        w.cheaptrick_coded_packed(x_packed, xo, fs, t, f0, fo, a.dims, cto, out=pkc[0])
        w.d4c_coded_packed(x_packed, xo, fs, t, f0, fo, sizes, d4o, out=pkc[1])

    def coded_padded():
        w._cheaptrick(True, x_pad, fs, t_pad, f0_pad, cto, lens, fl, a.dims, pdc[0])
        w._d4c(True, x_pad, fs, t_pad, f0_pad, sizes, d4o, lens, fl, pdc[1])

    legs = {"full_packed": full_packed, "full_padded": full_padded, "coded_packed": coded_packed,
            "coded_padded": coded_padded}
    for fn in legs.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in legs}
    in_use = {}
    for _ in range(3):   # three alternating rounds of a.steps steps per leg
        for k, fn in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / a.steps)
    # each leg's device-memory high-water: from a trimmed context (the library's scratch only grows within a call), the
    # memory in use after the leg, less what the resident arrays and context hold before it
    for k, fn in legs.items():
        w.trim()
        torch.cuda.synchronize()
        free0, total = torch.cuda.mem_get_info(dev)
        fn()
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info(dev)
        in_use[k] = {"before_gb": (total - free0) / 1e9, "after_gb": (total - free1) / 1e9,
                     "scratch_gb": (free0 - free1) / 1e9}
    w.synchronize()
    equal = {"full": True, "coded": True}
    for u in range(min(8, U)):
        a0, a1, f = int(fo[u]), int(fo[u + 1]), int(fl[u])
        equal["full"] = equal["full"] and all(torch.equal(p[a0:a1], q[u, :f]) for p, q in zip(pk, pd))
        equal["coded"] = equal["coded"] and torch.equal(pkc[0][a0:a1], pdc[0][u, :f]) and (
            n_ap == 0 or torch.equal(pkc[1][a0:a1], pdc[1][u, :f]))
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    out.update({"value": mean["full_packed"], "unit": "ms", "steps": a.steps, "warmup": a.warmup, "gpu": gpu_info(),
                "ms_per_call_pair": ms, "mean_ms": mean,
                "packed_over_padded_time": {"full": mean["full_packed"] / mean["full_padded"],
                                            "coded": mean["coded_packed"] / mean["coded_padded"]},
                "device_memory_per_leg": in_use,
                "check": {"utterances": min(8, U), "packed_equals_padded": equal}})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
