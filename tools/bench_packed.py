#!/usr/bin/env python
"""bench_packed.py -- the packed analysis chains against the padded ones on a corpus of mixed lengths.

A seeded corpus of N utterances (synthetic speech, tests/synth.py) whose lengths are drawn log-uniformly from
[1, 30] s, Harvest -> CheapTrick -> D4C with the default options.  Two pairs of calls on the same utterances, each pair
timed alternating, with the same steps and warm-up:

  device   world_b200_analyze_packed (full rows [F][bins])  vs  world_b200_analyze_batch_spectral_options
           (full rows [n][L][bins], L the longest utterance's frame count), DEVICE arrays
  host     world_b200_analyze_coded_host_packed  vs  world_b200_analyze_coded_host_spectral_options, 16-bit PCM in,
           coded rows out, HOST arrays

Reports each call's time, frames/s, device memory in use after each leg (cudaMemGetInfo), the output bytes, and the
host-to-device / device-to-host bytes of the host legs (counted from the shapes each call moves).  The first utterances
of each pair are compared bit for bit.  Prints ONE JSON line; writes nothing.  --count-only gives the byte counts
without a GPU.

  python tools/bench_packed.py [--utts 1024] [--fs 16000] [--steps 2] [--warmup 1] [--dims 40] [--count-only]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def corpus_lengths(n, fs, seed=7):
    rng = np.random.default_rng(seed)
    return [int(fs * s) for s in np.exp(rng.uniform(np.log(1.0), np.log(30.0), n))]


def frames(fs, n, frame_period=5.0):
    return int(1000.0 * n / fs / frame_period) + 1


def counts(lens, fs, bins, dims, n_ap):
    """Bytes of the padded and packed layouts: the device legs' full-row outputs, the host legs' transfers."""
    n, fl = len(lens), [frames(fs, v) for v in lens]
    L, F, S = max(fl), sum(fl), sum(lens)
    coded = (2 + dims + n_ap) * 8
    return {"frames_padded": n * L, "frames_packed": F,
            "device_output_bytes": {"padded": 2 * n * L * bins * 8, "packed": 2 * F * bins * 8},
            "host_h2d_bytes": {"padded": n * max(lens) * 2, "packed": S * 2},
            "host_d2h_bytes": {"padded": n * L * coded, "packed": F * coded},
            "padded_over_packed_samples": n * max(lens) / S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dims", type=int, default=40)
    ap.add_argument("--count-only", action="store_true")
    a = ap.parse_args()
    fs, U = a.fs, a.utts
    lens = corpus_lengths(U, fs)
    n_ap = max(0, int(min(15000.0, fs / 2.0 - 3000.0) / 3000.0))
    fft = 1 << int(np.ceil(np.log2(3.0 * fs / 71.0 + 1)))   # GetFFTSizeForCheapTrick at the default floor
    bins = fft // 2 + 1
    out = {"metric": "analysis frames/sec, Harvest+CheapTrick+D4C, packed batch of log-uniform 1-30 s utterances",
           "workload": f"{U} utterances, {fs // 1000} kHz synthetic speech, lengths log-uniform in [1, 30] s",
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
    x_pad = torch.zeros((U, M), dtype=torch.float64, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        xb = synth_batch(range(u0 + 1, u1 + 1), fs, max(lens[u0:u1]), device=dev)
        for u in range(u0, u1):
            x_pad[u, :lens[u]] = xb[u - u0, :lens[u]]
            x_packed[xo[u]:xo[u + 1]] = xb[u - u0, :lens[u]]
    ao = w.analysis_option(fs, F0_HARVEST)
    assert ao.cheaptrick.fft_size == fft
    fo = w.packed_frames(fs, xo, 5.0)
    F, fl = int(fo[-1]), np.diff(fo)
    L = int(fl.max())
    pk = [torch.zeros(F, dtype=torch.float64, device=dev) for _ in range(2)] + \
         [torch.zeros((F, bins), dtype=torch.float64, device=dev) for _ in range(2)]
    pd = [torch.zeros((U, L), dtype=torch.float64, device=dev) for _ in range(2)] + \
         [torch.zeros((U, L, bins), dtype=torch.float64, device=dev) for _ in range(2)]
    # 16-bit PCM for the host legs, packed and padded
    pcm_pad = np.zeros((U, M), dtype=np.int16)
    xh = x_pad.cpu().numpy()
    for u in range(U):
        pcm_pad[u, :lens[u]] = np.round(xh[u, :lens[u]] * 0.9 * 32767).astype(np.int16)
    pcm_packed = np.concatenate([pcm_pad[u, :lens[u]] for u in range(U)])
    del xh
    host_pk = [np.zeros(F), np.zeros(F), np.zeros((F, a.dims)), np.zeros((F, max(1, n_ap)))]
    host_pd = [np.zeros((U, L)), np.zeros((U, L)), np.zeros((U, L, a.dims)), np.zeros((U, L, max(1, n_ap)))]
    cto = [ao.cheaptrick] * U
    # both layouts' outputs stay allocated; the lanes' arenas and the host pipeline's each take up to the budget
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(max(2 << 30, free * 0.3)))

    def dev_packed():
        w.analyze_packed(x_packed, xo, fs, ao, time_axis=pk[0], f0=pk[1], spectrogram=pk[2], aperiodicity=pk[3])

    def dev_padded():
        w.analyze_batch(x_pad, fs, ao, x_lengths=lens, time_axis=pd[0], f0=pd[1], spectrogram=pd[2],
                        aperiodicity=pd[3], cheaptrick_options=cto)

    def host_packed():
        w.analyze_coded_host_packed(pcm_packed, 16, xo, fs, ao, a.dims, time_axis=host_pk[0], f0=host_pk[1],
                                    coded_sp=host_pk[2], coded_ap=host_pk[3])

    def host_padded():
        w.analyze_coded_host(pcm_pad, 16, fs, ao, a.dims, x_lengths=lens, time_axis=host_pd[0], f0=host_pd[1],
                             coded_sp=host_pd[2], coded_ap=host_pd[3], cheaptrick_options=cto)

    legs = {"device_packed": dev_packed, "device_padded": dev_padded, "host_packed": host_packed,
            "host_padded": host_padded}
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
            free, total = torch.cuda.mem_get_info(dev)
            in_use[k] = max(in_use.get(k, 0.0), (total - free) / 1e9)
    # the first utterances of each pair, bit for bit
    dev_packed(); dev_padded(); host_packed(); host_padded()
    torch.cuda.synchronize()
    equal = {"device": True, "host": True}
    for u in range(min(8, U)):
        a0, a1, f = int(fo[u]), int(fo[u + 1]), int(fl[u])
        equal["device"] = equal["device"] and all(torch.equal(p[a0:a1], q[u, :f]) for p, q in zip(pk, pd))
        equal["host"] = equal["host"] and all(np.array_equal(p[a0:a1], q[u, :f]) for p, q in zip(host_pk, host_pd))
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    out.update({"value": F / (mean["device_packed"] / 1e3), "unit": "frames/s", "steps": a.steps,
                "warmup": a.warmup, "gpu": gpu_info(), "ms_per_call": ms,
                "frames_per_s": {k: F / (v / 1e3) for k, v in mean.items()},
                "device_memory_in_use_gb_after_leg": in_use,
                "check": {"utterances": min(8, U), "packed_equals_padded": equal}})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
