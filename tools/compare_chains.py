"""Compares two builds of the library call by call: every analysis chain entry point, voice transformation, every
CheapTrick / D4C / StoneMask stage entry point, every synthesis entry point and modify on seeded ragged batches, with
each call's return code, launch count and outputs required to be identical byte for byte.  Meant for a refactor of the
chain, stage or synthesis drivers, with the parent commit's build as A and the change's as B (on the host emulation,
two tests/emu builds; on a GPU, two libworld_b200.so with --device).

    python tools/compare_chains.py A.so B.so [--device]

Analysis covers 8 and 16 kHz (16 kHz has one aperiodicity band, 8 kHz none), float64 and 16-bit PCM input, Harvest
and DIO, no options, per-utterance F0 options, per-utterance CheapTrick / D4C options with two FFT sizes, NULL
spectrogram / aperiodicity, transform with all three factors, and the host pipelines with small chunks (WB_HOST_CHUNK /
WB_HOST_SUB).  The stage calls cover 8, 16 and 44.1 kHz: one option, the same option for every utterance as lists, and
mixed options, into full and coded rows, and full rows wider than the largest size's bins.  Synthesis covers 8 and
16 kHz: full rows, coded rows to float64 and int16 on device and host arrays, with and without f0_scale /
spectral_ratio, and modify, on rows made by numpy (one full-length utterance's f0 is above 1.2 kHz, so its pass is laid
out again).  The stage calls and synthesis run at the default scratch budget and at the smallest one (several passes
and host chunks).  Prints the number of calls compared; exits 1 on the first difference."""
import argparse
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST, DioOption, HarvestOption, World, _ptr  # noqa: E402

DIMS = 20


def batch(fs, seed, n=5, seconds=0.3):
    rng = np.random.default_rng(seed)
    stride = int(fs * seconds)
    lens = [int(stride * f) for f in rng.uniform(0.6, 1.0, n)]
    lens[0] = stride
    t = np.arange(stride) / fs
    x = np.zeros((n, stride))
    for u, m in enumerate(lens):
        x[u, :m] = 0.4 * np.sin(2 * np.pi * rng.uniform(110, 260) * t[:m]) + 0.02 * rng.standard_normal(m)
    pcm = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    return x, pcm, lens


def f0_options(method, n):
    if method == F0_HARVEST:
        out = [HarvestOption() for _ in range(n)]
        for u, o in enumerate(out):
            o.f0_floor, o.f0_ceil, o.frame_period = 60.0 + 10 * u, 500.0 + 50 * u, 5.0
        return out
    out = [DioOption() for _ in range(n)]
    for u, o in enumerate(out):
        o.f0_floor, o.f0_ceil, o.channels_in_octave, o.allowed_range = 60.0 + 10 * u, 500.0 + 50 * u, 2.0, 0.1
        o.frame_period, o.speed = 5.0, 1
    return out


def calls(w, device):
    """(name, thunk) pairs; a thunk returns the outputs of one call on World w."""
    def arr(a):
        if not device:
            return a
        import torch
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    out = []
    for fs in (8000, 16000):
        x, pcm, lens = batch(fs, fs)
        n = len(lens)
        for method in (F0_HARVEST, F0_DIO_STONEMASK):
            ao = w.analysis_option(fs, method)
            tag = f"fs {fs} {'harvest' if method == F0_HARVEST else 'dio'}"
            small = ao.cheaptrick.fft_size
            cts, d4s = [w.cheaptrick_option(fs) for _ in range(n)], [w.d4c_option() for _ in range(n)]
            for u in range(0, n, 2):
                cts[u].fft_size = 2 * small
            for u, d in enumerate(d4s):
                d.threshold = 0.8 + 0.02 * u
            per_f0 = f0_options(method, n)
            f0_kw = [{}, {"harvest_options" if method == F0_HARVEST else "dio_options": per_f0}]
            for kw in f0_kw:
                name = f"{tag} {'per-utt F0' if kw else 'no options'}"
                out.append((f"analyze_batch {name}", lambda kw=kw, ao=ao, x=x, lens=lens, fs=fs:
                            w.analyze_batch(arr(x), fs, ao, x_lengths=lens, **kw)[:4]))
                out.append((f"analyze_host {name}", lambda kw=kw, ao=ao, x=x, lens=lens, fs=fs:
                            w.analyze_host(x, fs, ao, x_lengths=lens, **kw)[:4]))
                for nbit, xin in ((0, x), (16, pcm)):
                    out.append((f"analyze_coded_batch nbit {nbit} {name}",
                                lambda kw=kw, ao=ao, xin=xin, nbit=nbit, lens=lens, fs=fs:
                                w.analyze_coded_batch(arr(xin), nbit, fs, ao, DIMS, x_lengths=lens, **kw)[:4]))
                    out.append((f"analyze_coded_host nbit {nbit} {name}",
                                lambda kw=kw, ao=ao, xin=xin, nbit=nbit, lens=lens, fs=fs:
                                w.analyze_coded_host(xin, nbit, fs, ao, DIMS, x_lengths=lens, **kw)[:4]))
                    spec = dict(kw, cheaptrick_options=cts, d4c_options=d4s)
                    out.append((f"analyze_coded_batch nbit {nbit} {name} spectral options",
                                lambda spec=spec, ao=ao, xin=xin, nbit=nbit, lens=lens, fs=fs:
                                w.analyze_coded_batch(arr(xin), nbit, fs, ao, DIMS, x_lengths=lens, **spec)[:4]))
                    out.append((f"analyze_coded_host nbit {nbit} {name} spectral options",
                                lambda spec=spec, ao=ao, xin=xin, nbit=nbit, lens=lens, fs=fs:
                                w.analyze_coded_host(xin, nbit, fs, ao, DIMS, x_lengths=lens, **spec)[:4]))
                    ts = [1.0 + 0.1 * u for u in range(n)]
                    factors = dict(kw, f0_scale=[1.2] * n, spectral_ratio=[0.9 + 0.05 * u for u in range(n)],
                                   time_scale=ts)
                    out.append((f"transform nbit {nbit} {name}", lambda f=factors, ao=ao, xin=xin, nbit=nbit,
                                lens=lens, fs=fs: w.transform(arr(xin), nbit, fs, ao, x_lengths=lens, dtype="int16",
                                                              **f)))
                    out.append((f"transform_host nbit {nbit} {name}", lambda f=factors, ao=ao, xin=xin, nbit=nbit,
                                lens=lens, fs=fs: w.transform_host(xin, nbit, fs, ao, x_lengths=lens, **f)))
            # NULL spectrogram / aperiodicity: that stage is skipped
            L = max(w.frames(fs, m) for m in lens)
            for entry, host in (("analyze_coded_host", True), ("analyze_coded_batch", False)):
                for which in ("sp", "ap"):
                    def null_call(entry=entry, host=host, which=which, ao=ao, fs=fs, x=x, lens=lens, L=L):
                        mk = (lambda a: a) if host else arr
                        t, f0 = mk(np.zeros((n, L))), mk(np.zeros((n, L)))
                        sp = None if which == "sp" else mk(np.zeros((n, L, DIMS)))
                        ap = None if which == "ap" else mk(np.zeros((n, L, max(1, w.number_of_aperiodicities(fs)))))
                        xin = x if host else arr(x)
                        w._chain(entry, (_ptr(xin), 0, n, x.shape[1], (C.c_int * n)(*lens), fs, C.byref(ao)), n,
                                 None, None, (DIMS, _ptr(t), _ptr(f0), L, _ptr(sp), _ptr(ap)), device=not host)
                        return [a for a in (t, f0, sp, ap) if a is not None]
                    out.append((f"{entry} NULL {which} {tag}", null_call))
    return out


def to_np(a):
    if a is None:
        return np.zeros(0)
    if hasattr(a, "cpu"):
        return a.cpu().numpy()
    return np.asarray(a)


def synthesis_rows(fs, seed, n=5, fft=1024, seconds=1.5, fp=5.0):
    """f0, full rows and coded rows of n ragged utterances, all from numpy.  Utterance 1 is at 1.5 kHz and as long as
    the longest row: its 2,250 pulses exceed the 1,864 the pulse arrays are first sized for, so its pass is laid out
    again."""
    rng = np.random.default_rng(seed)
    Y, L, bins, n_ap = int(fs * seconds), int(seconds * 1000 / fp) + 1, fft // 2 + 1, 1 if fs == 16000 else 0
    ylens = [Y, Y] + [int(Y * f) for f in rng.uniform(0.6, 1.0, n - 2)]
    flens = [min(L, int(y / fs * 1000 / fp) + 2) for y in ylens]
    k = np.arange(bins) / bins
    f0, sp, ap = np.zeros((n, L)), np.ones((n, L, bins)), np.ones((n, L, bins))
    csp, cap = np.zeros((n, L, DIMS)), np.zeros((n, L, max(n_ap, 1)))
    for u, m in enumerate(flens):
        f0[u, :m] = np.where(rng.uniform(size=m) < 0.85, rng.uniform(90.0, 300.0), 0.0)
        sp[u, :m] = np.exp(-6.0 * k[None, :] + 0.3 * rng.normal(size=(m, 1))) * 1e-3
        ap[u, :m] = np.clip(k[None, :] ** 2 + 0.05 * rng.uniform(size=(m, bins)), 1e-3, 1 - 1e-12)
        csp[u, :m, 0] = -7.0 + 0.3 * rng.normal(size=m)
        csp[u, :m, 1:] = 0.3 * rng.normal(size=(m, DIMS - 1)) / np.arange(2, DIMS + 1)
        cap[u, :m] = -rng.uniform(1.0, 30.0, size=(m, cap.shape[2]))
    f0[1, :flens[1]] = 1500.0
    return f0, sp, ap, csp, (cap if n_ap else None), fft, fp, Y, flens, ylens


def synthesis_calls_at(w, arr, fs):
    """(name, thunk) pairs of the synthesis entry points and modify at one rate.  The thunks run after the whole list
    is built, so they read only this call's locals (and their own default arguments)."""
    f0, sp, ap, csp, cap, fft, fp, Y, fl, yl = synthesis_rows(fs, fs + 1)
    n, L = len(fl), f0.shape[1]
    factors = dict(f0_scale=[1.1 + 0.05 * u for u in range(n)], spectral_ratio=[0.9 + 0.05 * u for u in range(n)])
    out = [(f"synthesis fs {fs}", lambda: [w.synthesis(arr(f0), arr(sp), arr(ap), fft, fp, fs, Y, f0_lengths=fl,
                                                       y_lengths=yl)])]
    for dtype in ("float64", "int16"):
        for kw in ({}, factors):
            tag = f"fs {fs} {dtype}{' factors' if kw else ''}"
            out.append((f"synthesis_coded {tag}", lambda dtype=dtype, kw=kw: [w.synthesis_coded(
                arr(f0), arr(csp), arr(cap), fft, fp, fs, Y, f0_lengths=fl, y_lengths=yl, dtype=dtype, **kw)]))
            out.append((f"synthesis_coded_host {tag}", lambda dtype=dtype, kw=kw: [w.synthesis_coded_host(
                f0, csp, cap, fft, fp, fs, Y, f0_lengths=fl, y_lengths=yl, nbit=16 if dtype == "int16" else 0,
                **kw)]))

    # the plain entry points without factors, called directly
    def plain(entry, nbit, host):
        y = np.zeros((n, Y), dtype=np.int16 if nbit else np.float64)
        y = y if host else arr(y)
        src = (f0, csp, cap) if host else (arr(f0), arr(csp), arr(cap))
        head = (w._h, _ptr(src[0]), (C.c_int * n)(*fl), n, L, _ptr(src[1]), DIMS, _ptr(src[2]), fft, fp, fs,
                (C.c_int * n)(*yl), Y)
        rc = getattr(w.lib, entry)(*head, *((nbit,) if host else ()), _ptr(y))
        return [np.array([rc]), y]
    out.append((f"world_b200_synthesis_coded_batch fs {fs}", lambda: plain("world_b200_synthesis_coded_batch", 0,
                                                                             False)))
    out.append((f"world_b200_synthesis_coded_batch_pcm16 fs {fs}",
                lambda: plain("world_b200_synthesis_coded_batch_pcm16", 16, False)))
    for nbit in (0, 16):
        out.append((f"world_b200_synthesis_coded_host nbit {nbit} fs {fs}",
                    lambda nbit=nbit: plain("world_b200_synthesis_coded_host", nbit, True)))
    out.append((f"modify fs {fs}", lambda: list(w.modify(arr(f0.copy()), arr(sp.copy()), fs, fft, f0_lengths=fl,
                                                          **factors))))
    return out


def stage_calls_at(w, arr, fs):
    """(name, thunk) pairs of the nine CheapTrick, D4C and StoneMask stage entry points at one rate, on numpy rows: one
    option and mixed options (two FFT sizes, q1 / threshold per utterance), full and coded rows, and full rows wider
    than the largest size's bins (row_stride)."""
    x, _, lens = batch(fs, fs + 2)
    n, L = len(lens), w.frames(fs, x.shape[1])
    rng = np.random.default_rng(fs + 3)
    fl = [w.frames(fs, m) for m in lens]
    t = np.tile(np.arange(L) * 0.005, (n, 1))
    f0 = np.where(rng.uniform(size=(n, L)) < 0.8, rng.uniform(80.0, 300.0, size=(n, L)), 0.0)
    xd, td, fd = arr(x), arr(t), arr(f0)
    kw = dict(x_lengths=lens, f0_lengths=fl)
    ct = w.cheaptrick_option(fs)
    cts = [w.cheaptrick_option(fs) for _ in range(n)]
    for u, o in enumerate(cts):
        o.fft_size, o.q1 = ct.fft_size * (2 if u % 2 else 1), -0.15 + 0.02 * u
    d4s = [w.d4c_option() for _ in range(n)]
    for u, d in enumerate(d4s):
        d.threshold = 0.8 + 0.02 * u
    sizes = [o.fft_size for o in cts]
    wide = (n, L, max(sizes) // 2 + 8)
    out = [(f"stonemask fs {fs}", lambda: [w.stonemask(xd, fs, td, fd, **kw)])]
    for tag, opt, size, d4 in (("one option", ct, ct.fft_size, None), ("one option as lists", [ct] * n,
                                                                         [ct.fft_size] * n, [w.d4c_option()] * n),
                               ("mixed options", cts, sizes, d4s)):
        name = f"fs {fs} {tag}"
        out.append((f"cheaptrick {name}", lambda opt=opt: [w.cheaptrick(xd, fs, td, fd, opt, **kw)]))
        out.append((f"d4c {name}", lambda size=size, d4=d4: [w.d4c(xd, fs, td, fd, size, d4, **kw)]))
        out.append((f"cheaptrick_coded {name}", lambda opt=opt: [w.cheaptrick_coded(xd, fs, td, fd, DIMS, opt, **kw)]))
        out.append((f"d4c_coded {name}", lambda size=size, d4=d4: [w.d4c_coded(xd, fs, td, fd, size, d4, **kw)]))
        if isinstance(opt, list):
            out.append((f"cheaptrick row_stride {name}", lambda opt=opt: [
                w.cheaptrick(xd, fs, td, fd, opt, out=arr(np.full(wide, -1.0)), **kw)]))
            out.append((f"d4c row_stride {name}", lambda size=size, d4=d4: [
                w.d4c(xd, fs, td, fd, size, d4, out=arr(np.full(wide, -1.0)), **kw)]))
    return out


def stage_calls(w, device):
    """(name, thunk) pairs of the stage entry points at 8, 16 and 44.1 kHz."""
    def arr(a):
        if not device:
            return a
        import torch
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    return [c for fs in (8000, 16000, 44100) for c in stage_calls_at(w, arr, fs)]


def synthesis_calls(w, device):
    """(name, thunk) pairs of the synthesis entry points and modify at 8 and 16 kHz."""
    def arr(a):
        if not device or a is None:
            return a
        import torch
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    return synthesis_calls_at(w, arr, 8000) + synthesis_calls_at(w, arr, 16000)


def compare(worlds, lists, label):
    """Runs each pair of calls on the two builds; exits 1 on the first difference.  Returns the number compared."""
    compared = 0
    for (name, fa), (_, fb) in zip(*lists):
        res = []
        for w, fn in zip(worlds, (fa, fb)):
            before = w.launch_count()
            try:
                outs, err = fn(), None
            except Exception as e:   # both builds must fail the same way
                outs, err = (), str(e)
            w.synchronize()
            res.append((err, w.launch_count() - before, [to_np(o).tobytes() for o in outs]))
        if res[0] != res[1]:
            print(f"DIFFERENT: {name} ({label}): errors {res[0][0]!r} / {res[1][0]!r}, launches "
                  f"{res[0][1]} / {res[1][1]}, outputs equal: {res[0][2] == res[1][2]}")
            sys.exit(1)
        if res[0][0]:
            print(f"note: both builds raised for {name}: {res[0][0]}")
        compared += 1
    return compared


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--device", action="store_true", help="CUDA builds, device arrays as torch tensors")
    args = ap.parse_args()
    mod = None if args.device else "numpy"
    libs = (args.lib_a, args.lib_b)
    worlds = [World(lib_path=p, array_module=mod or "torch") for p in libs]
    compared = 0
    for chunks in ((None, None), ("2", "1")):
        for k, v in zip(("WB_HOST_CHUNK", "WB_HOST_SUB"), chunks):
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        compared += compare(worlds, [calls(w, args.device) for w in worlds], f"chunks {chunks}")
    for k in ("WB_HOST_CHUNK", "WB_HOST_SUB"):
        os.environ.pop(k, None)
    # the stage calls and synthesis at the default scratch budget, then at the smallest one (64 MB: several passes and
    # host chunks)
    small = [World(lib_path=p, array_module=mod or "torch") for p in libs]
    for w in small:
        w.set_scratch_budget(64 << 20)
    for ws, label in ((worlds, "default budget"), (small, "64 MB budget")):
        compared += compare(ws, [stage_calls(w, args.device) for w in ws], label)
        compared += compare(ws, [synthesis_calls(w, args.device) for w in ws], label)
    print(f"{compared} calls compared, all identical (return codes, launch counts, output bytes)")


if __name__ == "__main__":
    main()
