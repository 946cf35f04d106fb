#!/usr/bin/env python
"""bench_coded_batch.py -- the coded chain on device arrays (world_b200_analyze_coded_batch*), PCM in, coded rows out.

Two workloads of BASELINE.json, on synthetic 16 kHz speech (tests/synth.py, quantised to int16), Harvest ->
CheapTrick -> D4C, 60 coded dimensions:

  --mode single   config 3 (1024 x 10 s) on one GPU.  Three legs on the same batch, alternating in one session:
                    coded      analyze_coded_batch on int16 rows -> time axis, f0, coded envelope, coded aperiodicity
                    coded_f64  analyze_coded_batch on the same samples as float64 rows (what the PCM conversion costs)
                    full_rows  analyze_batch on the float64 rows -> full spectrogram / aperiodicity
                  Reported: frames/s of each leg (CUDA events; median over rounds after warm-up), and the device
                  memory each call needed -- free memory (torch.cuda.mem_get_info) before the call minus free memory
                  after it, with the library's pooled and arena memory and torch's cache given back first; the input
                  rows are resident before and are reported apart.
  --mode gather   config 5 in full (8192 x 5 s) over the ranks of torchrun (1, 2, 4 or 8 GPUs, 8192 / ranks utterances
                  each): analyze_coded_batch_allgather, every rank ending with the coded rows of the whole corpus.
                  Afterwards every rank recomputes the first utterance of every other rank's shard on its own GPU and
                  checks the gathered rows bit for bit.

Prints ONE JSON line (rank 0); writes nothing.

  python tools/bench_coded_batch.py --mode single [--utts 1024] [--seconds 10] [--steps 2] [--warmup 1] [--rounds 5]
  torchrun --nproc-per-node G tools/bench_coded_batch.py --mode gather [--corpus 8192] [--seconds 5]
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


def int16_batch(torch, seeds, fs, n, dev):
    """synthetic rows quantised to int16 on the device (64 utterances per generator call)"""
    from synth import synth_batch
    seeds = list(seeds)
    x = torch.empty((len(seeds), n), dtype=torch.int16, device=dev)
    for u0 in range(0, len(seeds), 64):
        u1 = min(len(seeds), u0 + 64)
        xs = synth_batch(seeds[u0:u1], fs, n, device=dev)
        x[u0:u1] = torch.clamp(torch.round(xs * 32768.0), -32768, 32767).to(torch.int16)
    return x


def timed(torch, legs, steps, warmup, rounds):
    """ms per call of every leg: warm-up, then `rounds` alternating rounds of `steps` calls per leg; median"""
    for fn in legs.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in legs}
    for _ in range(rounds):
        for k, fn in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / steps)
    return ms


def single(a):
    import torch
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_f0_ranges import gpu_info

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, n, U = a.fs, int(a.fs * a.seconds), a.utts
    x16 = int16_batch(torch, range(1, U + 1), fs, n, dev)
    xd = x16.to(torch.float64) / 32768.0
    ao = w.analysis_option(fs, F0_HARVEST)
    L = w.frames(fs, n, ao.harvest.frame_period)
    bins = ao.cheaptrick.fft_size // 2 + 1
    n_ap = w.number_of_aperiodicities(fs)
    w.set_scratch_budget(int(a.scratch_gb * (1 << 30)))

    def coded(outs=None, x=x16, nbit=16):
        kw = {} if outs is None else dict(time_axis=outs[0], f0=outs[1], coded_sp=outs[2], coded_ap=outs[3])
        return w.analyze_coded_batch(x, nbit, fs, ao, DIMS, **kw)

    def full_rows(outs=None):
        kw = {} if outs is None else dict(time_axis=outs[0], f0=outs[1], spectrogram=outs[2], aperiodicity=outs[3])
        return w.analyze_batch(xd, fs, ao, **kw)

    # device memory one call needs: outputs, scratch arena, lane buffers (inputs are resident already)
    need = {}
    for k, fn in (("coded", coded), ("full_rows", full_rows)):
        w.trim()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0, _ = torch.cuda.mem_get_info(dev)
        outs = fn()
        w.synchronize()
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info(dev)
        need[k] = free0 - free1
        del outs
    w.trim()
    torch.cuda.empty_cache()
    # timed legs write into resident outputs
    oc = coded()
    of = full_rows()
    w.synchronize()
    od = coded(x=xd, nbit=0)
    w.synchronize()
    same = {"time_axis": bool(torch.equal(oc[0], of[0])), "f0": bool(torch.equal(oc[1], of[1])),
            "coded rows, int16 vs float64 input": all(bool(torch.equal(p, q)) for p, q in zip(oc[:4], od[:4]))}
    legs = {"coded": lambda: coded(oc[:4]), "coded_f64": lambda: coded(od[:4], xd, 0),
            "full_rows": lambda: full_rows(of[:4])}
    sampler = ClockSampler(0)
    sampler.start()
    ms = timed(torch, legs, a.steps, a.warmup, a.rounds)
    clocks = sampler.stop()
    frames = U * L
    med = {k: statistics.median(v) for k, v in ms.items()}
    gb = 1e9
    out = {"metric": "analysis frames/sec, Harvest+CheapTrick+D4C on device arrays: coded rows from int16 vs full rows "
                     "from float64",
           "value": frames / (med["coded"] / 1e3), "unit": "frames/s",
           "workload": f"{U}x{a.seconds:g}s synthetic {fs // 1000} kHz batch (BASELINE config 3), one GPU, "
                       f"{DIMS} coded dimensions + {n_ap} aperiodicity band(s)",
           "frames_per_s": {k: frames / (v / 1e3) for k, v in med.items()},
           "ms_per_call_median": med, "ms_per_call_rounds": ms, "steps": a.steps, "warmup": a.warmup,
           "rounds": a.rounds,
           "device_gb_needed_by_call": {k: v / gb for k, v in need.items()},
           "input_gb": {"coded (int16)": x16.numel() * 2 / gb, "full_rows (float64)": xd.numel() * 8 / gb},
           "output_gb": {"coded": U * L * (2 + DIMS + n_ap) * 8 / gb, "full_rows": U * L * (2 + 2 * bins) * 8 / gb},
           "bit_identical_between_legs": same,
           "scratch_budget_gb": a.scratch_gb, "gpu": gpu_info(), "clocks_during_timing": clocks}
    print(json.dumps(out), flush=True)


def gather(a):
    import torch
    import torch.distributed as dist
    from world_b200.api import World, F0_HARVEST
    from bench import ClockSampler
    from bench_f0_ranges import gpu_info

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if a.corpus % world:
        raise SystemExit(f"--corpus {a.corpus} does not split evenly over {world} ranks")
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")

    def quiet(fn):   # NCCL prints its banner on stdout; the one JSON line must stay alone there
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(2, 1)
        try:
            return fn()
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved)

    if world > 1:
        quiet(lambda: dist.init_process_group("nccl", device_id=dev))
    w = World(device=local)
    idt = torch.zeros(128, dtype=torch.uint8, device=dev)
    if rank == 0:
        idt.copy_(torch.frombuffer(bytearray(w.comm_unique_id()), dtype=torch.uint8))
    if world > 1:
        dist.broadcast(idt, 0)
    quiet(lambda: w.comm_init(world, rank, bytes(idt.cpu().numpy().tobytes())))

    fs, n, U = a.fs, int(a.fs * a.seconds), a.corpus // world
    x16 = int16_batch(torch, range(rank * U + 1, rank * U + U + 1), fs, n, dev)
    ao = w.analysis_option(fs, F0_HARVEST)
    L = w.frames(fs, n, ao.harvest.frame_period)
    n_ap = w.number_of_aperiodicities(fs)
    N = world * U
    outs = [torch.zeros((N, L), dtype=torch.float64, device=dev), torch.zeros((N, L), dtype=torch.float64, device=dev),
            torch.zeros((N, L, DIMS), dtype=torch.float64, device=dev),
            torch.zeros((N, L, max(1, n_ap)), dtype=torch.float64, device=dev)]
    free, _ = torch.cuda.mem_get_info(dev)
    w.set_scratch_budget(int(min(96 << 30, max(2 << 30, free * 0.45))))

    def step():
        w.analyze_coded_batch_allgather(x16, 16, fs, ao, DIMS, *outs)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(a.warmup):
        step()
    w.synchronize()
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms = []
    for _ in range(a.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        e0.record()
        for _ in range(a.steps):
            step()
        e1.record()
        w.synchronize()
        barrier()
        t = e0.elapsed_time(e1) / a.steps
        if world > 1:
            tt = torch.tensor([t], dtype=torch.float64, device=dev)
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            t = float(tt.item())
        ms.append(t)
    clocks = sampler.stop() if rank == 0 else None
    # the first utterance of every other rank's shard, recomputed here, against the gathered rows
    ok, checked = True, []
    for r in range(world):
        if r == rank:
            continue
        xr = int16_batch(torch, range(r * U + 1, r * U + min(U, 64) + 1), fs, n, dev)[:1].contiguous()
        mine = w.analyze_coded_batch(xr, 16, fs, ao, DIMS)
        w.synchronize()
        ok = ok and all(torch.equal(m, g[r * U:r * U + 1]) for m, g in zip(mine[:4], outs))
        checked.append(r * U)
    flags = torch.tensor([1 if ok else 0, len(checked)], dtype=torch.int64, device=dev)
    if world > 1:
        dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    voiced = float((outs[1] > 0).double().mean())
    med = statistics.median(ms)
    if rank == 0:
        gb = 1e9
        out = {"metric": "analysis frames/sec, Harvest+CheapTrick+D4C from int16, coded rows all-gathered on every rank",
               "value": N * L / (med / 1e3), "unit": "frames/s",
               "workload": f"{N}x{a.seconds:g}s synthetic {fs // 1000} kHz corpus (BASELINE config 5), {world} GPU(s), "
                           f"{U} utterances per GPU, {DIMS} coded dimensions + {n_ap} aperiodicity band(s)",
               "ms_per_call_median": med, "ms_per_call_rounds": ms, "steps": a.steps, "warmup": a.warmup,
               "rounds": a.rounds, "gathered_gb_per_rank": sum(o.numel() for o in outs) * 8 / gb,
               "gather_check": {"bit_identical_on_every_rank": bool(flags[0].item()),
                                "other_ranks_checked_per_rank": int(flags[1].item())},
               "voiced_share": voiced, "gpu": gpu_info(), "clocks_during_timing": clocks}
        print(json.dumps(out), flush=True)
    w.comm_destroy()
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", required=True, choices=["single", "gather"])
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--utts", type=int, default=1024, help="single: utterances in the batch")
    ap.add_argument("--corpus", type=int, default=8192, help="gather: utterances over all ranks")
    ap.add_argument("--seconds", type=float, default=None, help="utterance length (default 10 single, 5 gather)")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scratch-gb", type=float, default=24.0, help="single: the library's scratch budget")
    a = ap.parse_args()
    if a.seconds is None:
        a.seconds = 10.0 if a.mode == "single" else 5.0
    single(a) if a.mode == "single" else gather(a)


if __name__ == "__main__":
    main()
