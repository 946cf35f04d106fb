#!/usr/bin/env python
"""bench_transform_packed.py -- the packed voice transformation against the padded one on a speed-perturbed corpus.

The corpus of bench_packed.py (corpus_lengths): N seeded utterances of synthetic speech with lengths log-uniform in
[1, 30] s at 16 kHz, as int16; Harvest, CheapTrick and D4C with the default options.  Each utterance gets a seeded
f0_scale in [0.8, 1.25], spectral_ratio in [0.9, 1.1] and time_scale from {0.9, 1.0, 1.1} (speed perturbation), and
the output is int16.  Four legs on the same utterances, timed alternately with CUDA events after warm-up (median):
  1. World.transform_packed on device arrays (world_b200_transform_packed);
  2. World.transform on the same utterances padded to the longest (world_b200_transform_batch);
  3. World.transform_host_packed from pinned host memory into a pinned host array;
  4. World.transform_host, padded, from pinned host memory into a pinned host array.
For each: ms per call, and the device memory the call needs: free memory (torch.cuda.mem_get_info) before and after
one call from a trimmed context and an emptied torch cache (the library keeps its arenas and pools at their peak, so
the difference is the call's high-water mark).  The host legs' PCIe bytes are counted from the shapes they move.  Leg 1
is compared with leg 2 utterance by utterance, and leg 3 with leg 1, bit for bit.  The card's name, power limit and SM
clocks are read in the same run.

Prints ONE JSON line; writes nothing.  --count-only prints the counted bytes without a GPU.

  python tools/bench_transform_packed.py [--utts 512] [--fs 16000] [--warmup 1] [--rounds 3] [--count-only]
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

from bench_packed import corpus_lengths, frames  # noqa: E402

FRAME_PERIOD = 5.0


def factors(n, seed=11):
    """Seeded per-utterance f0_scale, spectral_ratio and time_scale (speed perturbation: 0.9, 1.0 or 1.1)."""
    rng = np.random.default_rng(seed)
    return (rng.uniform(0.8, 1.25, n).tolist(), rng.uniform(0.9, 1.1, n).tolist(),
            rng.choice([0.9, 1.0, 1.1], n).tolist())


def out_samples(fs, n, time_scale):
    """world_b200_transform_samples: the demo's y_length at frame period FRAME_PERIOD * time_scale (one product)."""
    return int((frames(fs, n, FRAME_PERIOD) - 1) * (FRAME_PERIOD * time_scale) / 1000.0 * fs) + 1


def counts(lens, y_lens):
    """PCIe bytes of the host legs (int16 in and out) and the padding of the padded layout."""
    n, S, Y = len(lens), sum(lens), sum(y_lens)
    return {"host_h2d_bytes": {"padded": n * max(lens) * 2, "packed": S * 2},
            "host_d2h_bytes": {"padded": n * max(y_lens) * 2, "packed": Y * 2},
            "padded_over_packed_samples": {"in": n * max(lens) / S, "out": n * max(y_lens) / Y}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=512)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--count-only", action="store_true")
    a = ap.parse_args()
    fs, U = a.fs, a.utts
    lens = corpus_lengths(U, fs)
    scale, ratio, tscale = factors(U)
    y_lens = [out_samples(fs, n, t) for n, t in zip(lens, tscale)]
    out = {"metric": "voice transformation of a speed-perturbed corpus of log-uniform 1-30 s int16 utterances, seconds "
                     "of audio per second (transform_packed on device arrays)",
           "unit": "audio s/s",
           "workload": f"{U} utterances, {fs // 1000} kHz synthetic speech int16, lengths log-uniform in [1, 30] s, "
                       "Harvest, per-utterance f0_scale in [0.8, 1.25], spectral_ratio in [0.9, 1.1], time_scale in "
                       "{0.9, 1.0, 1.1}, int16 out",
           "counted": counts(lens, y_lens)}
    if a.count_only:
        print(json.dumps(out), flush=True)
        return
    import torch
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_coded_batch import int16_batch, timed
    from bench_f0_ranges import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("bench_transform_packed.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    S, M = sum(lens), max(lens)
    xo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x_pad = torch.zeros((U, M), dtype=torch.int16, device=dev)
    x_packed = torch.empty(S, dtype=torch.int16, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        xb = int16_batch(torch, range(u0 + 1, u1 + 1), fs, max(lens[u0:u1]), dev)
        for u in range(u0, u1):
            x_pad[u, :lens[u]] = xb[u - u0, :lens[u]]
            x_packed[xo[u]:xo[u + 1]] = xb[u - u0, :lens[u]]
        del xb
    x_pad_host, x_packed_host = x_pad.cpu().pin_memory(), x_packed.cpu().pin_memory()
    ao = w.analysis_option(fs, F0_HARVEST)
    yo = w.transform_packed_samples(fs, xo, FRAME_PERIOD, tscale)
    assert list(np.diff(yo)) == y_lens
    Y = int(yo[-1])
    y_packed_host = torch.zeros(Y, dtype=torch.int16).pin_memory()
    y_pad_host = torch.zeros((U, max(y_lens)), dtype=torch.int16).pin_memory()
    kw = dict(f0_scale=scale, spectral_ratio=ratio, time_scale=tscale, dtype="int16")
    res = {}

    def leg1():
        res[1] = w.transform_packed(x_packed, 16, xo, fs, ao, **kw)[0]

    def leg2():
        res[2] = w.transform(x_pad, 16, fs, ao, x_lengths=lens, **kw)[0]

    def leg3():
        w.transform_host_packed(x_packed_host, 16, xo, fs, ao, out=y_packed_host, **kw)
        res[3] = y_packed_host

    def leg4():
        w.transform_host(x_pad_host, 16, fs, ao, x_lengths=lens, out=y_pad_host, **kw)
        res[4] = y_pad_host

    legs = {"1_transform_packed": leg1, "2_transform_padded": leg2, "3_transform_host_packed_pinned": leg3,
            "4_transform_host_padded_pinned": leg4}
    mem_gb = {}
    for k, fn in legs.items():   # one call each from a trimmed context: the memory high-water, and the first warm-up
        res.clear()
        w.synchronize()
        w.trim()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0, _ = torch.cuda.mem_get_info()
        fn()
        w.synchronize()
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info()
        mem_gb[k] = (free0 - free1) / 1e9
    res.clear()
    sampler = ClockSampler(0)
    sampler.start()
    ms = timed(torch, {k: (lambda fn=fn: (fn(), w.synchronize())) for k, fn in legs.items()}, 1, a.warmup, a.rounds)
    clocks = sampler.stop()
    torch.cuda.synchronize()
    med = {k: statistics.median(v) for k, v in ms.items()}
    # every utterance, bit for bit: leg 1 against leg 2, leg 3 against leg 1 (the legs' last timed outputs)
    y1, y2 = res[1], res[2]
    eq12 = all(torch.equal(y1[int(yo[u]):int(yo[u + 1])], y2[u, :y_lens[u]]) for u in range(U))
    eq31 = bool(torch.equal(res[3], y1.cpu()))
    audio_s = S / fs
    out.update({
        "value": audio_s / (med["1_transform_packed"] / 1e3),
        "ms_median": med, "ms_rounds": ms,
        "audio_s_per_s": {k: audio_s / (v / 1e3) for k, v in med.items()},
        "padded_over_packed_ms": {"device": med["2_transform_padded"] / med["1_transform_packed"],
                                  "host": med["4_transform_host_padded_pinned"] /
                                  med["3_transform_host_packed_pinned"]},
        "device_memory_high_water_gb": mem_gb,
        "leg1_equals_leg2_per_utterance_bitwise": bool(eq12), "leg3_equals_leg1_bitwise": eq31,
        "utterances": U, "audio_s": audio_s, "warmup": a.warmup, "rounds": a.rounds,
        "clocks_during_timing": clocks, "gpu": gpu_info()})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
