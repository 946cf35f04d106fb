#!/usr/bin/env python
"""bench_modify_curves.py -- pitch and formant curves (one factor per frame) against one factor per utterance.

The corpus of bench_packed.py (corpus_lengths): N seeded utterances of synthetic speech with lengths log-uniform in
[1, 30] s at 16 kHz, Harvest, CheapTrick and D4C with the default options (fft_size 1024), rows from analyze_packed.
Each utterance gets the seeded f0_scale, spectral_ratio and time_scale of bench_transform_packed.py.  Two curves per
frame are built from them: constant (curve[f] = the utterance's factor) and smooth random (the factor times a slow
seeded sinusoid, about +-10 % on f0 and +-5 % on the ratio).

Modification, on the packed rows in place; every leg first restores the rows from a saved copy, and a copy-only leg
gives that share:
  modify_packed (factors; host-planned stretch tables), modify_curves_packed on constant curves and on smooth curves.
Transformation, float64 samples on device in, int16 out:
  transform_packed (factors), transform_packed_curves on constant curves and on smooth curves.
Legs are timed alternately with CUDA events after warm-up (median ms per call).  On constant curves the curve calls
are compared with the factor calls bit for bit (rows, and every output sample).  The card's name, power limit and SM
clocks are read in the same run.

Prints ONE JSON line; writes nothing.

  python tools/bench_modify_curves.py [--utts 512] [--fs 16000] [--warmup 1] [--rounds 3] [--steps 3]
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

from bench_packed import corpus_lengths  # noqa: E402
from bench_transform_packed import factors  # noqa: E402

FRAME_PERIOD = 5.0


def curves(fo, scale, ratio, seed=13):
    """(constant f0, constant ratio, smooth f0, smooth ratio) curves [F] over the frame offsets fo."""
    rng = np.random.default_rng(seed)
    F = int(fo[-1])
    cf, cr, sf, sr = (np.empty(F) for _ in range(4))
    for u in range(len(scale)):
        a, b = int(fo[u]), int(fo[u + 1])
        t = np.arange(b - a) * FRAME_PERIOD / 1000.0
        cf[a:b], cr[a:b] = scale[u], ratio[u]
        sf[a:b] = scale[u] * np.exp(0.1 * np.sin(2 * np.pi * rng.uniform(0.2, 2.0) * t + rng.uniform(0, 6.3)))
        sr[a:b] = ratio[u] * np.exp(0.05 * np.sin(2 * np.pi * rng.uniform(0.1, 1.0) * t + rng.uniform(0, 6.3)))
    return cf, cr, sf, sr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=512)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3, help="modification calls per timed round")
    a = ap.parse_args()

    import torch
    from world_b200.api import World, F0_HARVEST
    from synth import synth_batch
    from bench import ClockSampler
    from bench_coded_batch import timed
    from bench_f0_ranges import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("bench_modify_curves.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    w = World(device=0)
    fs, U = a.fs, a.utts
    lens = corpus_lengths(U, fs)
    S = sum(lens)
    xo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x = torch.empty(S, dtype=torch.float64, device=dev)
    for u0 in range(0, U, 32):
        u1 = min(U, u0 + 32)
        xb = synth_batch(range(u0 + 1, u1 + 1), fs, max(lens[u0:u1]), device=dev)
        for u in range(u0, u1):
            x[xo[u]:xo[u + 1]] = xb[u - u0, :lens[u]]
        del xb
    ao = w.analysis_option(fs, F0_HARVEST)
    fft = ao.cheaptrick.fft_size
    _, f0, sp, _, fo = w.analyze_packed(x, xo, fs, ao)
    w.synchronize()
    assert np.array_equal(fo, w.packed_frames(fs, xo, FRAME_PERIOD))
    F = int(fo[-1])
    scale, ratio, tscale = factors(U)
    cf, cr, sf, sr = (torch.from_numpy(c).to(dev) for c in curves(fo, scale, ratio))
    sizes = [fft] * U
    f0_base, sp_base = f0.clone(), sp.clone()
    outs = {}

    def restore():
        f0.copy_(f0_base)
        sp.copy_(sp_base)

    def mod_factors():
        restore()
        w.modify_packed(f0, sp, fo, fs, fft_size=sizes, f0_scale=scale, spectral_ratio=ratio)

    def mod_curves(c_f, c_r):
        restore()
        w.modify_curves_packed(f0, sp, fo, fs, fft_size=sizes, f0_curve=c_f, spectral_ratio_curve=c_r)

    # bit for bit on constant curves
    mod_factors()
    want_f0, want_sp = f0.clone(), sp.clone()
    mod_curves(cf, cr)
    w.synchronize()
    mod_equal = bool(torch.equal(f0, want_f0) and torch.equal(sp, want_sp))
    del want_f0, want_sp
    mod_legs = {"copy_only": restore, "modify_packed_factors": mod_factors,
                "modify_curves_packed_constant": lambda: mod_curves(cf, cr),
                "modify_curves_packed_smooth": lambda: mod_curves(sf, sr)}
    sampler = ClockSampler(0)
    sampler.start()
    mod_ms = timed(torch, {k: (lambda fn=fn: (fn(), w.synchronize())) for k, fn in mod_legs.items()}, a.steps,
                   a.warmup, a.rounds)
    del f0, sp, f0_base, sp_base
    w.trim()
    torch.cuda.empty_cache()

    kw = dict(time_scale=tscale, dtype="int16")
    tr_legs = {
        "transform_packed_factors": lambda: outs.__setitem__("f", w.transform_packed(
            x, 0, xo, fs, ao, f0_scale=scale, spectral_ratio=ratio, **kw)[0]),
        "transform_packed_curves_constant": lambda: outs.__setitem__("c", w.transform_packed_curves(
            x, 0, xo, fs, ao, f0_curve=cf, spectral_ratio_curve=cr, **kw)[0]),
        "transform_packed_curves_smooth": lambda: outs.__setitem__("s", w.transform_packed_curves(
            x, 0, xo, fs, ao, f0_curve=sf, spectral_ratio_curve=sr, **kw)[0]),
    }
    tr_ms = timed(torch, {k: (lambda fn=fn: (fn(), w.synchronize())) for k, fn in tr_legs.items()}, 1, a.warmup,
                  a.rounds)
    clocks = sampler.stop()
    torch.cuda.synchronize()
    tr_equal = bool(torch.equal(outs["f"], outs["c"]))
    med_mod = {k: statistics.median(v) for k, v in mod_ms.items()}
    med_tr = {k: statistics.median(v) for k, v in tr_ms.items()}
    audio_s = S / fs
    out = {"metric": "pitch and formant curves against per-utterance factors: modify_curves_packed and "
                     "transform_packed_curves, ms per call (median)",
           "unit": "ms",
           "workload": f"{U} utterances, {fs // 1000} kHz synthetic speech, lengths log-uniform in [1, 30] s, Harvest, "
                       f"fft_size {fft}, {F} frames; factors f0_scale in [0.8, 1.25], spectral_ratio in [0.9, 1.1], "
                       "time_scale in {0.9, 1.0, 1.1}; curves constant or smooth random; transform int16 out",
           "value": med_mod["modify_curves_packed_smooth"],
           "modify_ms_median": med_mod, "modify_ms_rounds": mod_ms,
           "modify_ms_without_copy": {k: v - med_mod["copy_only"] for k, v in med_mod.items() if k != "copy_only"},
           "transform_ms_median": med_tr, "transform_ms_rounds": tr_ms,
           "transform_audio_s_per_s": {k: audio_s / (v / 1e3) for k, v in med_tr.items()},
           "modify_constant_curves_equal_factors_bitwise": mod_equal,
           "transform_constant_curves_equal_factors_bitwise": tr_equal,
           "frames": F, "utterances": U, "audio_s": audio_s, "warmup": a.warmup, "rounds": a.rounds,
           "steps": a.steps, "clocks_during_timing": clocks, "gpu": gpu_info()}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
