#!/usr/bin/env python
"""bench_synthesis_host.py -- Synthesis from coded rows for a caller holding HOST memory: the pipelined host call
against copying up, synthesising and copying down in series.

Features are built once as tools/bench_synthesis.py builds them (analyze_coded_batch on the int16 synthetic batch:
Harvest -> CheapTrick -> D4C, 60 coded dimensions) and copied into pinned host memory.  Four legs, alternating in one
session; the first three go from pinned host rows to a pinned host waveform:

  host_pcm16   synthesis_coded_host, nbit 16: upload / synthesis / int16 download pipelined over utterance chunks
  host_f64     synthesis_coded_host, nbit 0: the same with the float64 waveform
  serial_f64   the status quo: copy f0 + coded rows up, synthesis_coded, copy the float64 waveform down, all on one
               stream
  device_only_f64  for reference, synthesis_coded on device-resident rows with the waveform left on the device: the
               compute the three legs above share, without PCIe

Reported: ms per call (host clock from call to results in host memory, after a device synchronisation; median over
rounds after warm-up) and output samples/s of each leg; the bytes each leg moves over PCIe; the WB_HOST_TRACE timeline
of one host_pcm16 call (a separate call after the timing); host_pcm16 == quantise(serial_f64) and host_f64 ==
serial_f64 (quantise = wavwrite's rule, trunc(y * 32767) clamped to int16); the GPU's name, power limit and clocks
during the timing.

Prints ONE JSON line; writes nothing in the tree (the trace goes through a temporary file).

  python tools/bench_synthesis_host.py [--utts 1024] [--seconds 10] [--fs 16000] [--warmup 1] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

DIMS = 60


def traced(fn):
    """fn() with WB_HOST_TRACE=1; returns the library's trace lines (stderr captured at the file descriptor)."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        os.environ["WB_HOST_TRACE"] = "1"
        try:
            fn()
        finally:
            del os.environ["WB_HOST_TRACE"]
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return [l.rstrip("\n") for l in f if l.startswith("[wb trace]")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scratch-gb", type=float, default=24.0, help="the library's scratch budget")
    a = ap.parse_args()

    import torch
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_coded_batch import int16_batch
    from bench_f0_ranges import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("bench_synthesis_host.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x16 = int16_batch(torch, range(1, U + 1), fs, n, dev)
    ao = w.analysis_option(fs, F0_HARVEST)
    fft, fp = ao.cheaptrick.fft_size, ao.harvest.frame_period
    w.set_scratch_budget(int(a.scratch_gb * (1 << 30)))
    _, f0_d, csp_d, cap_d, fl = w.analyze_coded_batch(x16, 16, fs, ao, DIMS)
    n_ap = w.number_of_aperiodicities(fs)
    w.synchronize()
    del x16
    f0 = f0_d.cpu().pin_memory()
    csp = csp_d.cpu().pin_memory()
    cap = cap_d.cpu().pin_memory() if n_ap > 0 else None
    del f0_d, csp_d, cap_d
    w.trim()
    torch.cuda.empty_cache()
    out16 = torch.empty((U, n), dtype=torch.int16).pin_memory()
    out64 = torch.empty((U, n), dtype=torch.float64).pin_memory()
    out_serial = torch.empty((U, n), dtype=torch.float64).pin_memory()

    def host_pcm16():
        w.synthesis_coded_host(f0, csp, cap, fft, fp, fs, n, nbit=16, out=out16)

    def host_f64():
        w.synthesis_coded_host(f0, csp, cap, fft, fp, fs, n, nbit=0, out=out64)

    def serial_f64():
        F = f0.to(dev, non_blocking=True)
        S = csp.to(dev, non_blocking=True)
        A = cap.to(dev, non_blocking=True) if cap is not None else None
        y = w.synthesis_coded(F, S, A, fft, fp, fs, n)
        out_serial.copy_(y, non_blocking=True)
        torch.cuda.current_stream().synchronize()

    F_res = f0.to(dev)
    S_res = csp.to(dev)
    A_res = cap.to(dev) if cap is not None else None

    def device_only():   # synthesis_coded on inputs already on the device, output left there: no PCIe at all
        w.synthesis_coded(F_res, S_res, A_res, fft, fp, fs, n)
        torch.cuda.current_stream().synchronize()

    legs = {"host_pcm16": host_pcm16, "host_f64": host_f64, "serial_f64": serial_f64, "device_only_f64": device_only}
    for fn in legs.values():
        for _ in range(a.warmup):
            fn()
    sampler = ClockSampler(0)
    sampler.start()
    ms = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, fn in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3)
    clocks = sampler.stop()
    med = {k: statistics.median(v) for k, v in ms.items()}

    # the outputs of the last round
    q = torch.clamp(torch.trunc(out_serial * 32767), -32768, 32767).to(torch.int16)
    checks = {"host_pcm16_equals_quantised_serial_f64": bool(torch.equal(out16, q)),
              "host_f64_equals_serial_f64": bool(torch.equal(out64, out_serial))}
    del q
    trace = traced(host_pcm16)

    gb = 1e9
    in_bytes = (f0.numel() + csp.numel() + (cap.numel() if cap is not None else 0)) * 8
    samples = U * n
    out = {"metric": "host-to-host synthesis from coded rows: pipelined synthesis_coded_host (int16) vs serial "
                     "upload + synthesis_coded + float64 download",
           "value": samples / (med["host_pcm16"] / 1e3), "unit": "samples/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch, Harvest features, fft {fft}, "
                       f"{DIMS} coded dimensions + {n_ap} aperiodicity band(s), pinned host buffers",
           "samples_per_s": {k: samples / (v / 1e3) for k, v in med.items()},
           "ms_per_call_median": med, "ms_per_call_rounds": ms, "warmup": a.warmup, "rounds": a.rounds,
           "pcie_gb": {"host_pcm16": {"h2d": in_bytes / gb, "d2h": samples * 2 / gb},
                       "host_f64": {"h2d": in_bytes / gb, "d2h": samples * 8 / gb},
                       "serial_f64": {"h2d": in_bytes / gb, "d2h": samples * 8 / gb},
                       "device_only_f64": {"h2d": 0.0, "d2h": 0.0}},
           **checks, "voiced_share": float((f0 > 0).double().mean()),
           "trace_host_pcm16": trace,
           "scratch_budget_gb": a.scratch_gb, "gpu": gpu_info(), "clocks_during_timing": clocks}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
