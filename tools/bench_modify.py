#!/usr/bin/env python
"""bench_modify.py -- F0 scaling and formant shift on device arrays.

  (a) world_b200_modify_batch on config-3-shaped rows: f0 [1024][2001] and envelopes [1024][2001][513] (fft 1024),
      every frame valid, a different (scale, ratio) per utterance (six distinct ratios, shrink and stretch).  Timed
      with CUDA events, median over rounds after warm-up, next to a torch copy of the envelope array in the same run.  The
      compulsory bytes are 16 per bin (the row is read and written once) plus 16 per frame of f0.  The call works in
      place, so every timed call stretches the previous result again; the ratios keep every query inside the source
      axis (no extrapolation), so the values stay within their first range.
  (b) synthesis_coded_batch against synthesis_coded_batch_modified on the same batch (default 256 x 10 s of synthetic
      16 kHz speech, Harvest features, 60 coded dimensions), alternating, reported as the modified call's overhead.
The card's name, power limit and clocks are read in the same run.

Prints ONE JSON line; writes nothing.

  python tools/bench_modify.py [--utts 1024] [--frames 2001] [--fft 1024] [--syn-utts 256] [--seconds 10] [--rounds 7]
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

DIMS = 60
RATIOS = (0.8, 0.9, 1.0, 1.1, 1.2, 1.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--frames", type=int, default=2001)
    ap.add_argument("--fft", type=int, default=1024)
    ap.add_argument("--syn-utts", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()

    import torch
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_coded_batch import int16_batch, timed
    from bench_f0_ranges import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("bench_modify.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    gb = 1e9

    # ---- (a) modify_batch against a copy of the same bytes
    U, L, fft, fs = a.utts, a.frames, a.fft, a.fs
    bins = fft // 2 + 1
    g = torch.Generator(device=dev).manual_seed(7)
    sp = torch.exp(torch.randn((U, L, bins), dtype=torch.float64, device=dev, generator=g) - 8.0)
    f0 = torch.where(torch.rand((U, L), device=dev, generator=g) < 0.7, 100.0 + 200.0 * torch.rand((U, L), device=dev,
                     generator=g), 0.0).to(torch.float64)
    ratios = [RATIOS[u % len(RATIOS)] for u in range(U)]
    scales = [0.99 if u % 2 else 1.01 for u in range(U)]
    copy_dst = torch.empty_like(sp)
    legs = {"modify_batch": lambda: w.modify(f0, sp, fs, fft, f0_scale=scales, spectral_ratio=ratios),
            "torch_copy": lambda: copy_dst.copy_(sp)}
    sampler = ClockSampler(0)
    sampler.start()
    ms_a = timed(torch, legs, 1, a.warmup, a.rounds)
    clocks_a = sampler.stop()
    finite = bool(torch.isfinite(sp).all())
    med_a = {k: statistics.median(v) for k, v in ms_a.items()}
    moved = {"modify_batch": U * L * bins * 16 + U * L * 16, "torch_copy": U * L * bins * 16}
    del sp, copy_dst, f0
    torch.cuda.empty_cache()

    # ---- (b) the modified synthesis against the plain one
    S, n = a.syn_utts, int(a.fs * a.seconds)
    x16 = int16_batch(torch, range(1, S + 1), fs, n, dev)
    ao = w.analysis_option(fs, F0_HARVEST)
    sfft, fp = ao.cheaptrick.fft_size, ao.harvest.frame_period
    _, f0s, csp, cap, fl = w.analyze_coded_batch(x16, 16, fs, ao, DIMS)
    cap = cap if w.number_of_aperiodicities(fs) > 0 else None
    w.synchronize()
    del x16
    s_scales = [0.8 + 0.45 * (u % 10) / 9 for u in range(S)]
    s_ratios = [0.9 + 0.25 * (u % 7) / 6 for u in range(S)]
    legs_b = {"synthesis_coded_batch": lambda: w.synthesis_coded(f0s, csp, cap, sfft, fp, fs, n),
              "synthesis_coded_batch_modified": lambda: w.synthesis_coded(f0s, csp, cap, sfft, fp, fs, n,
                                                                          f0_scale=s_scales, spectral_ratio=s_ratios)}
    sampler = ClockSampler(0)
    sampler.start()
    ms_b = timed(torch, legs_b, 1, 1, a.rounds)
    clocks_b = sampler.stop()
    med_b = {k: statistics.median(v) for k, v in ms_b.items()}
    overhead = 100.0 * (med_b["synthesis_coded_batch_modified"] / med_b["synthesis_coded_batch"] - 1.0)

    out = {"metric": "world_b200_modify_batch compulsory bytes per second on config-3-shaped rows",
           "value": moved["modify_batch"] / (med_a["modify_batch"] / 1e3) / gb, "unit": "GB/s",
           "modify": {"shape": [U, L, bins], "fft_size": fft, "distinct_ratios": len(set(ratios)),
                      "gb_moved": {k: v / gb for k, v in moved.items()}, "ms_median": med_a, "ms_rounds": ms_a,
                      "gb_per_s": {k: moved[k] / (v / 1e3) / gb for k, v in med_a.items()},
                      "share_of_copy_bandwidth": (moved["modify_batch"] / med_a["modify_batch"])
                                                 / (moved["torch_copy"] / med_a["torch_copy"]),
                      "rows_stay_finite": finite,
                      "clocks_during_timing": clocks_a},
           "synthesis": {"workload": f"{S}x{a.seconds:g}s synthetic {fs // 1000} kHz, Harvest features, fft {sfft}, "
                                     f"{DIMS} coded dimensions, a different scale / ratio per utterance",
                         "ms_median": med_b, "ms_rounds": ms_b, "modified_overhead_pct": overhead,
                         "clocks_during_timing": clocks_b},
           "warmup": a.warmup, "rounds": a.rounds, "gpu": gpu_info()}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
