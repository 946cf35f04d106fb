#!/usr/bin/env python
"""bench_transform.py -- voice transformation, PCM in and PCM out, on the config-3 shape.

Default batch: 1024 x 10 s of synthetic 16 kHz speech as int16, Harvest, CheapTrick fft 1024, f0_scale 1.3,
spectral_ratio 0.9, time_scale 1, int16 out.  Three legs, timed alternately with CUDA events after warm-up (median):
  (a) World.transform on device arrays (world_b200_transform_batch);
  (b) the stepwise full-row chain for the same batch: pcm_to_double -> analyze_batch -> modify -> synthesis, then the
      pcm16 rule in torch;
  (c) World.transform_host from pinned host memory into a pinned host array (world_b200_transform_host).
For each: ms per call, seconds of audio per second, and the device memory the call needs: free memory
(torch.cuda.mem_get_info) before and after one call from a trimmed context and an emptied torch cache.  The library
allocates with cudaMalloc and keeps its arenas and pooled buffers at their peak, and torch keeps its cache, so the
difference is the call's high-water mark.  (a) against (b) and (c) against (a) are compared bit for bit on the timed
batch.  The card's name, power limit and SM clocks are read in the same run.

Prints ONE JSON line; writes nothing.

  python tools/bench_transform.py [--utts 1024] [--seconds 10] [--fs 16000] [--warmup 1] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

F0_SCALE, SPECTRAL_RATIO = 1.3, 0.9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()

    import torch
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_coded_batch import int16_batch, timed
    from bench_f0_ranges import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("bench_transform.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    U, fs, n = a.utts, a.fs, int(a.fs * a.seconds)
    x16 = int16_batch(torch, range(1, U + 1), fs, n, dev)
    x16_host = x16.cpu().pin_memory()
    ao = w.analysis_option(fs, F0_HARVEST)
    fft, fp = ao.cheaptrick.fft_size, ao.harvest.frame_period
    y_len = w.transform_samples(fs, n, fp)
    y_host = torch.zeros((U, y_len), dtype=torch.int16).pin_memory()
    out = {}

    def leg_a():
        out["a"] = w.transform(x16, 16, fs, ao, f0_scale=F0_SCALE, spectral_ratio=SPECTRAL_RATIO, dtype="int16")[0]

    def leg_b():
        x = w.pcm_to_double(x16, 16)
        _, f0, sp, ap_, fl = w.analyze_batch(x, fs, ao)
        del x
        w.modify(f0, sp, fs, fft, f0_scale=F0_SCALE, spectral_ratio=SPECTRAL_RATIO, f0_lengths=fl)
        y = w.synthesis(f0, sp, ap_, fft, fp, fs, y_len, f0_lengths=fl)
        del f0, sp, ap_
        out["b"] = torch.clamp(torch.trunc(y * 32767.0), -32768, 32767).to(torch.int16)

    def leg_c():
        w.transform_host(x16_host, 16, fs, ao, f0_scale=F0_SCALE, spectral_ratio=SPECTRAL_RATIO, dtype="int16",
                         out=y_host)
        out["c"] = y_host

    legs = {"a_transform": leg_a, "b_stepwise": leg_b, "c_transform_host_pinned": leg_c}
    mem_gb = {}
    for k, fn in legs.items():   # one call each from a trimmed context: the memory high-water, and the first warm-up
        out.clear()
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
    out.clear()
    sampler = ClockSampler(0)
    sampler.start()
    ms = timed(torch, {k: (lambda fn=fn: (fn(), w.synchronize())) for k, fn in legs.items()}, 1, a.warmup, a.rounds)
    clocks = sampler.stop()
    med = {k: statistics.median(v) for k, v in ms.items()}
    audio_s = U * a.seconds
    result = {
        "metric": "voice transformation of config-3-shaped int16 batches, seconds of audio per second (transform on "
                  "device arrays)",
        "value": audio_s / (med["a_transform"] / 1e3), "unit": "audio s/s",
        "workload": f"{U} x {a.seconds:g} s synthetic {fs // 1000} kHz int16, Harvest, fft {fft}, f0_scale {F0_SCALE}, "
                    f"spectral_ratio {SPECTRAL_RATIO}, time_scale 1, int16 out ({y_len} samples per utterance)",
        "ms_median": med, "ms_rounds": ms,
        "audio_s_per_s": {k: audio_s / (v / 1e3) for k, v in med.items()},
        "speedup_a_over_b": med["b_stepwise"] / med["a_transform"],
        "device_memory_high_water_gb": mem_gb,
        "a_equals_b_bitwise": bool(torch.equal(out["a"], out["b"])),
        "c_equals_a_bitwise": bool(torch.equal(out["c"], out["a"].cpu())),
        "warmup": a.warmup, "rounds": a.rounds, "clocks_during_timing": clocks, "gpu": gpu_info()}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
