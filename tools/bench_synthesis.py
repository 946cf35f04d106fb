#!/usr/bin/env python
"""bench_synthesis.py -- Synthesis on device arrays: from coded rows in one call, against the two-step path.

Features are built once with analyze_coded_batch (Harvest -> CheapTrick -> D4C, 60 coded dimensions) on the synthetic
speech of tests/synth.py (quantised to int16, as tools/bench_coded_batch.py does).  Three legs on that batch,
alternating in one session:

  coded       synthesis_coded: f0 + coded rows in, waveform out; the rows are decoded chunk by chunk inside the call
  two_step    decode_spectral_envelope + decode_aperiodicity over the whole batch, then synthesis
  decoded     synthesis on rows that are already decoded (the pure synthesis cost)

Reported: ms per call (CUDA events; median over rounds after warm-up) and output samples/s of each leg; the per-kernel
profile of one call of each leg (world_b200_profile_report, in a run of its own after the timing); the device memory
the coded and two-step calls needed on top of their inputs -- free memory (torch.cuda.mem_get_info) before the call
minus free memory after it, with the library's arena and torch's cache given back first; torch.equal of the coded and
two-step outputs; the GPU's name, power limit and clocks during the timing.

Prints ONE JSON line; writes nothing.

  python tools/bench_synthesis.py [--utts 256] [--seconds 10] [--fs 16000] [--steps 1] [--warmup 1] [--rounds 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scratch-gb", type=float, default=24.0, help="the library's scratch budget")
    a = ap.parse_args()

    import torch
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_coded_batch import int16_batch, timed
    from bench_f0_ranges import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("bench_synthesis.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x16 = int16_batch(torch, range(1, U + 1), fs, n, dev)
    ao = w.analysis_option(fs, F0_HARVEST)
    fft, fp = ao.cheaptrick.fft_size, ao.harvest.frame_period
    w.set_scratch_budget(int(a.scratch_gb * (1 << 30)))
    _, f0, csp, cap, fl = w.analyze_coded_batch(x16, 16, fs, ao, DIMS)
    n_ap = w.number_of_aperiodicities(fs)
    cap = cap if n_ap > 0 else None
    w.synchronize()
    del x16
    L = f0.shape[1]

    def coded():
        return w.synthesis_coded(f0, csp, cap, fft, fp, fs, n)

    def decode():
        sp = w.decode_spectral_envelope(csp, fs, fft, DIMS)
        ap_rows = w.decode_aperiodicity(cap if cap is not None else torch.zeros((U, L, 1), dtype=torch.float64,
                                                                                device=dev), fs, fft)
        return sp, ap_rows

    def two_step():
        sp, ap_rows = decode()
        return w.synthesis(f0, sp, ap_rows, fft, fp, fs, n)

    # device memory one call needs beyond its (resident) inputs: output, decoded rows, scratch arena
    need = {}
    for k, fn in (("coded", coded), ("two_step", two_step)):
        w.trim()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0, _ = torch.cuda.mem_get_info(dev)
        y = fn()
        w.synchronize()
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info(dev)
        need[k] = free0 - free1
        del y
    w.trim()
    torch.cuda.empty_cache()

    ya, yb = coded(), two_step()
    w.synchronize()
    equal = bool(torch.equal(ya, yb))
    del ya, yb
    sp_d, ap_d = decode()
    w.synchronize()
    legs = {"coded": coded, "two_step": two_step,
            "decoded": lambda: w.synthesis(f0, sp_d, ap_d, fft, fp, fs, n)}
    sampler = ClockSampler(0)
    sampler.start()
    ms = timed(torch, legs, a.steps, a.warmup, a.rounds)
    clocks = sampler.stop()
    med = {k: statistics.median(v) for k, v in ms.items()}

    profile = {}
    for k, fn in legs.items():
        w.profile(True)
        fn()
        profile[k] = w.profile_report()
        w.profile(False)
    gb = 1e9
    samples = U * n
    out = {"metric": "synthesis output samples/sec on device arrays: coded rows in one call vs decode + synthesis",
           "value": samples / (med["coded"] / 1e3), "unit": "samples/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch, Harvest features, fft {fft}, "
                       f"{DIMS} coded dimensions + {n_ap} aperiodicity band(s)",
           "samples_per_s": {k: samples / (v / 1e3) for k, v in med.items()},
           "ms_per_call_median": med, "ms_per_call_rounds": ms, "steps": a.steps, "warmup": a.warmup,
           "rounds": a.rounds,
           "device_gb_needed_by_call": {k: v / gb for k, v in need.items()},
           "input_gb": {"coded": (f0.numel() + csp.numel() + (cap.numel() if cap is not None else 0)) * 8 / gb,
                        "decoded rows": (sp_d.numel() + ap_d.numel()) * 8 / gb},
           "output_gb": U * n * 8 / gb,
           "coded_equals_two_step": equal, "voiced_share": float((f0 > 0).double().mean()),
           "profile_one_call": profile,
           "scratch_budget_gb": a.scratch_gb, "gpu": gpu_info(), "clocks_during_timing": clocks}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
