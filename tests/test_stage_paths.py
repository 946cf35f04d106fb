"""The stage drivers' rarely taken paths against the reference: scratch chunks (u0 > 0), D4C's slow body kernel on
both sides of its split, rates above 48 kHz, and Synthesis over rates, frame periods, ragged batches and f0 up to
2.4 kHz.  Each check is written once and runs on the host emulation (CPU suite) and on the CUDA library (-m gpu).
Tolerances are the project's: 1e-6 relative for f0 / spectrogram / aperiodicity, a bit-exact time axis, no V/UV
flip, and 1e-9 of the waveform peak for Synthesis."""
import numpy as np
import pytest

from test_parity_common import TOL, assert_close, assert_close_signed, make, to_np
from refworld import rel_err

SMALL_BUDGET = 64 << 20      # the smallest scratch budget world_b200_set_scratch_budget accepts


def _with_budget(world, nbytes):
    """A second context of the same kind as `world` (same library, same device) with its own scratch budget, so
    the session's shared context keeps its default."""
    from world_b200.api import World
    w = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    w.set_scratch_budget(nbytes)
    return w


def _same(a, b, what):
    a, b = to_np(a), to_np(b)
    assert a.shape == b.shape and np.array_equal(a, b), f"{what}: chunked result differs from the one-pass result"


def _contours(rng, frames, L):
    """A 1 ms time axis, shifted by 0.3 ms more in each utterance (a row read at another utterance's offset must not
    give the same frames), and a random f0 (70-400 Hz, a fifth of the frames unvoiced) for each utterance."""
    t, f = np.zeros((len(frames), L)), np.zeros((len(frames), L))
    for u, n in enumerate(frames):
        t[u, :n] = np.arange(n) / 1000.0 + 0.0003 * u
        f[u, :n] = np.where(rng.uniform(size=n) < 0.8, rng.uniform(70.0, 400.0, size=n), 0.0)
    return t, f


# ---------------------------------------------------------------- 1. scratch chunks (set_scratch_budget)
def check_chunks_cheaptrick(world, ref):
    from synth import synth_batch
    fs, n_utt, secs = 16000, 10, 2.5
    # cheaptrick_run: per utterance (fft_size + bins) * 4 B of draws per frame * max frames + 8 B * f_stride + 64
    #   = 1537 * 4 * 2501 + 8 * 2501 + 64 = 15,396,220 B  -> 4 per 64 MB pass; 10 utterances -> passes of 4, 4, 2
    n = int(secs * fs)
    lens = [n - 1601 * u for u in range(n_utt)]
    frames = [int(1000.0 * l / fs) + 1 for l in lens]
    x = synth_batch(range(201, 201 + n_utt), fs, n).numpy()
    t, f = _contours(np.random.default_rng(1), frames, frames[0])
    xb, tb, fb = make(world, x), make(world, t), make(world, f)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs = []
        for w in (world, small):
            opt = w.cheaptrick_option(fs)
            outs.append((w.cheaptrick(xb, fs, tb, fb, opt, x_lengths=lens, f0_lengths=frames),
                         w.cheaptrick_coded(xb, fs, tb, fb, 40, opt, x_lengths=lens, f0_lengths=frames)))
            w.synchronize()
    finally:
        small.close()
    (sp, csp), (sp_s, csp_s) = outs
    _same(sp_s, sp, "CheapTrick")
    _same(csp_s, csp, "CheapTrick + CodeSpectralEnvelope")
    u = n_utt - 1                                          # in the last, shorter pass
    xu, tu, fu = x[u, :lens[u]], t[u, :frames[u]], f[u, :frames[u]]
    want = ref.cheaptrick(xu, fs, tu, fu)
    assert_close(to_np(sp_s)[u, :frames[u]], want, "CheapTrick, last chunk")
    assert_close_signed(to_np(csp_s)[u, :frames[u]], ref.code_spectral_envelope(want, fs, 1024, 40),
                        "coded CheapTrick, last chunk")
    return max(rel_err(to_np(sp_s)[u, :frames[u]], want).max(), 0.0)


def check_chunks_d4c(world, ref):
    from synth import synth_batch
    worst = 0.0
    # d4c_run: per utterance (max_a + max_b) * 4 B of draws per frame * max frames + 28 B * f_stride + 64
    #   16 kHz:    (1201 + 4089) * 4 * 1501 + 28 * 1501 + 64 = 31,803,252 B -> 2 per pass; 5 -> passes of 2, 2, 1
    #   22.05 kHz: (1655 + 5631) * 4 * 1001 + 28 * 1001 + 64 = 29,201,236 B -> 2 per pass; 5 -> passes of 2, 2, 1
    #   (D4C + CodeAperiodicity: nothing is coded below 22.05 kHz, so the fused kernel runs at 22.05 kHz)
    for fs, secs, n_utt, coded in ((16000, 1.5, 5, False), (22050, 1.0, 5, True)):
        n = int(secs * fs)
        lens = [n - int(0.07 * fs) * u for u in range(n_utt)]
        frames = [int(1000.0 * l / fs) + 1 for l in lens]
        x = synth_batch(range(301, 301 + n_utt), fs, n).numpy()
        t, f = _contours(np.random.default_rng(fs), frames, frames[0])
        xb, tb, fb = make(world, x), make(world, t), make(world, f)
        fft = world.cheaptrick_option(fs).fft_size
        small = _with_budget(world, SMALL_BUDGET)
        try:
            outs = []
            for w in (world, small):
                if coded:
                    outs.append(w.d4c_coded(xb, fs, tb, fb, fft, x_lengths=lens, f0_lengths=frames))
                else:
                    outs.append(w.d4c(xb, fs, tb, fb, fft, x_lengths=lens, f0_lengths=frames))
                w.synchronize()
        finally:
            small.close()
        _same(outs[1], outs[0], f"D4C{' + CodeAperiodicity' if coded else ''} fs {fs}")
        u = n_utt - 1
        xu, tu, fu = x[u, :lens[u]], t[u, :frames[u]], f[u, :frames[u]]
        want = ref.d4c(xu, fs, tu, fu, fft)
        got = to_np(outs[1])[u, :frames[u]]
        if coded:
            assert ref.number_of_aperiodicities(fs) == got.shape[1] == 2
            assert_close_signed(got, ref.code_aperiodicity(want, fs, fft), f"coded D4C fs {fs}, last chunk")
        else:
            assert_close(got, want, f"D4C fs {fs}, last chunk")
            worst = max(worst, rel_err(got, want).max())
    return worst


def check_chunks_harvest_and_chain(world, ref):
    """Harvest alone, and analyze_batch (F0_HARVEST) whose two lanes each get half the budget."""
    from synth import synth_batch
    from world_b200 import api
    fs, n_utt, secs = 16000, 5, 3.0
    # harvest_run: per utterance (per_utt_bytes at 16 kHz, default option) 31,657,160 B for 3 s -> 2 per 64 MB pass;
    #   5 utterances -> passes of 2, 2, 1.  Each lane of analyze_batch runs at 32 MB: one utterance per pass.
    n = int(secs * fs)
    lens = [n - 2203 * u for u in range(n_utt)]
    x = synth_batch(range(401, 401 + n_utt), fs, n).numpy()
    xb = make(world, x)
    opt = world.analysis_option(fs, api.F0_HARVEST)
    t, f0, fl = world.harvest(xb, fs, opt.harvest, x_lengths=lens)
    sp = world.cheaptrick(xb, fs, t, f0, opt.cheaptrick, x_lengths=lens, f0_lengths=fl)
    ap = world.d4c(xb, fs, t, f0, opt.cheaptrick.fft_size, x_lengths=lens, f0_lengths=fl)
    world.synchronize()
    small = _with_budget(world, SMALL_BUDGET)
    try:
        t_s, f0_s, _ = small.harvest(xb, fs, opt.harvest, x_lengths=lens)
        chain = small.analyze_batch(xb, fs, opt, x_lengths=lens)
        small.synchronize()
    finally:
        small.close()
    _same(t_s, t, "Harvest time axis")
    _same(f0_s, f0, "Harvest f0")
    for got, want, name in zip(chain[:4], (t, f0, sp, ap), ("time axis", "f0", "spectrogram", "aperiodicity")):
        got, want = to_np(got), to_np(want)
        for u in range(n_utt):
            assert np.array_equal(got[u, :fl[u]], want[u, :fl[u]]), f"analyze_batch {name} utt {u} (64 MB budget)"
    u = n_utt - 1
    tr, fr = ref.harvest(x[u, :lens[u]], fs)
    g = to_np(f0_s)[u, :fl[u]]
    assert np.array_equal(to_np(t_s)[u, :fl[u]], tr)
    assert not ((g > 0) != (fr > 0)).any()
    assert_close(g, fr, "Harvest f0, last chunk")
    return rel_err(g, fr).max()


def check_chunks_dio_stonemask(world, ref):
    from synth import synth_batch
    fs, n_utt, secs = 16000, 7, 10.0
    # dio_run: per utterance (per_utt at 16 kHz, default option) 20,920,328 B for 10 s -> 3 per pass; 7 -> 3, 3, 1.
    # stonemask_run keeps no per-utterance scratch (one pass below 65535 utterances): it must not care either.
    n = int(secs * fs)
    lens = [n - 4001 * u for u in range(n_utt)]
    x = synth_batch(range(501, 501 + n_utt), fs, n).numpy()
    xb = make(world, x)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs = []
        for w in (world, small):
            t, f0, fl = w.dio(xb, fs, x_lengths=lens)
            sm = w.stonemask(xb, fs, t, f0, x_lengths=lens, f0_lengths=fl)
            w.synchronize()
            outs.append((t, f0, sm))
    finally:
        small.close()
    for a, b, name in zip(outs[1], outs[0], ("DIO time axis", "DIO f0", "StoneMask f0")):
        _same(a, b, name)
    u = n_utt - 1
    t, f0, sm = (to_np(a)[u, :fl[u]] for a in outs[1])
    tr, fr = ref.dio(x[u, :lens[u]], fs)
    smr = ref.stonemask(x[u, :lens[u]], fs, tr, fr)
    assert np.array_equal(t, tr)
    assert not ((f0 > 0) != (fr > 0)).any()
    assert_close(f0, fr, "DIO f0, last chunk")
    assert_close(sm, smr, "StoneMask f0, last chunk")
    return max(rel_err(f0, fr).max(), rel_err(sm, smr).max())


def check_chunks_synthesis(world, ref):
    fs, n_utt, secs, fft = 16000, 7, 2.0, 1024
    # world_b200_synthesis_batch: per utterance y_stride * 16 + cap * (20 + fft_size * 8) + (y + 8) * 4 + 4096 with
    #   cap = 2 s * 1200 + 64 pulses: 20,878,496 B -> 3 per pass; 7 -> passes of 3, 3, 1 if no pass had more pulses.
    #   Utterance 4 runs at 2 kHz over 26,652 samples (about 3,330 pulses, 28 MB at that cap -> 2 per pass), so the
    #   passes are 3 (utterances 0-2), 2 (3-4, laid out again for utterance 4's count) and 2 (5-6).
    rng = np.random.default_rng(17)
    n = int(secs * fs)
    ylens = [n - 1337 * u for u in range(n_utt)]
    L = int(secs * 200) + 1
    flens = [L - 7 * u for u in range(n_utt)]
    bins = fft // 2 + 1
    f0 = np.zeros((n_utt, L)); sp = np.ones((n_utt, L, bins)); ap = np.ones((n_utt, L, bins))
    k = np.arange(bins) / bins
    for u in range(n_utt):
        m = flens[u]
        f0[u, :m] = np.where(rng.uniform(size=m) < 0.85, rng.uniform(90.0, 300.0) * (1 + 0.2 * np.sin(np.arange(m) / 30.0)), 0.0)
        sp[u, :m] = np.exp(-6.0 * k[None, :] + 0.3 * rng.normal(size=(m, 1))) * 1e-3
        ap[u, :m] = np.clip(k[None, :] ** 2 + 0.05 * rng.uniform(size=(m, bins)), 1e-3, 1 - 1e-12)
    f0[4, :flens[4]] = 2000.0
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs = []
        for w in (world, small):
            outs.append(w.synthesis(make(w, f0), make(w, sp), make(w, ap), fft, 5.0, fs, n, f0_lengths=flens,
                                    y_lengths=ylens))
            w.synchronize()
    finally:
        small.close()
    _same(outs[1], outs[0], "Synthesis")
    worst = 0.0
    for u in (4, n_utt - 1):
        yr = ref.synthesis(f0[u, :flens[u]], sp[u, :flens[u]], ap[u, :flens[u]], fft, 5.0, fs, ylens[u])
        e = np.abs(to_np(outs[1])[u, :ylens[u]] - yr).max() / np.abs(yr).max()
        assert e <= 1e-9, f"Synthesis utt {u}: {e:.2e} of the peak"
        worst = max(worst, e)
    return worst


CHUNK_CHECKS = {"cheaptrick": check_chunks_cheaptrick, "d4c": check_chunks_d4c,
                "harvest_and_chain": check_chunks_harvest_and_chain, "dio_stonemask": check_chunks_dio_stonemask,
                "synthesis": check_chunks_synthesis}


# ---------------------------------------------------------------- 2. D4C's fast / slow body split
def f0_ramp(fs, lo=30.0, hi=110.0):
    """lo..hi Hz with consecutive ratio-4 windows (~4 * 1.5 * fs / f0 samples) at most 2 samples apart:
    f0[i+1] - f0[i] <= f0[i]^2 / (2 fs)."""
    f = [lo]
    while f[-1] < hi:
        f.append(f[-1] + f[-1] * f[-1] / (2.0 * fs))
    return np.array(f)


def check_d4c_split(world, ref, fs):
    """Every window length on both sides of the fast / slow split, in a batch of two (the second utterance has
    the ramp reversed and shorter, so its list entries carry an utterance offset); f0 below D4C's 47 Hz floor and
    0 Hz frames included.  More than 2 x 132 slow frames: each persistent CTA takes several."""
    from synth import synth_batch
    ramp = f0_ramp(fs)
    fa = ramp.copy(); fa[::97] = 0.0
    fb = ramp[::-1][len(ramp) // 10:].copy(); fb[5::89] = 0.0
    frames = [len(fa), len(fb)]
    L = frames[0]
    # the slow side starts near 54 Hz at 16 kHz and 75 Hz at 48 kHz
    assert sum(int(((c > 0) & (c < 54.0)).sum()) for c in (fa, fb)) > 2 * 132
    lens = [int((frames[u] - 1) * fs / 1000.0) + fs // 50 for u in range(2)]
    x = synth_batch([601, 602], fs, lens[0]).numpy()
    t = np.zeros((2, L)); f = np.zeros((2, L))
    for u, c in enumerate((fa, fb)):
        t[u, :len(c)] = np.arange(len(c)) / 1000.0
        f[u, :len(c)] = c
    xb, tb, fbd = make(world, x), make(world, t), make(world, f)
    opt = world.cheaptrick_option(fs)
    fft = opt.fft_size
    dims = 40
    sp = world.cheaptrick(xb, fs, tb, fbd, opt, x_lengths=lens, f0_lengths=frames)
    ap = world.d4c(xb, fs, tb, fbd, fft, x_lengths=lens, f0_lengths=frames)
    csp = world.cheaptrick_coded(xb, fs, tb, fbd, dims, opt, x_lengths=lens, f0_lengths=frames)
    cap = world.d4c_coded(xb, fs, tb, fbd, fft, x_lengths=lens, f0_lengths=frames)
    world.synchronize()
    n_ap = ref.number_of_aperiodicities(fs)
    worst = 0.0
    for u in range(2):
        m = frames[u]
        xu, tu, fu = x[u, :lens[u]], t[u, :m], f[u, :m]
        spr = ref.cheaptrick(xu, fs, tu, fu)
        apr = ref.d4c(xu, fs, tu, fu, fft)
        assert_close(to_np(sp)[u, :m], spr, f"CheapTrick fs {fs} utt {u}")
        assert_close(to_np(ap)[u, :m], apr, f"D4C fs {fs} utt {u}")
        assert_close_signed(to_np(csp)[u, :m], ref.code_spectral_envelope(spr, fs, fft, dims),
                            f"coded CheapTrick fs {fs} utt {u}")
        if n_ap > 0:
            assert_close_signed(to_np(cap)[u, :m], ref.code_aperiodicity(apr, fs, fft), f"coded D4C fs {fs} utt {u}")
        worst = max(worst, rel_err(to_np(ap)[u, :m], apr).max(), rel_err(to_np(sp)[u, :m], spr).max())
    return worst


# ---------------------------------------------------------------- 3. 88.2 and 96 kHz
def check_high_rate_chain(world, ref, fs, lens):
    """Harvest -> CheapTrick (fft 4096) -> D4C (d_fft 8192: every frame on the list kernel) against the reference's
    own chain, on a ragged batch; the same chain through analyze_batch and analyze_host (F0_HARVEST); the fused coded
    kernels and the codec (5 aperiodicity bands)."""
    from synth import synth_batch
    from world_b200 import api
    n_utt = len(lens)
    x = synth_batch(range(701, 701 + n_utt), fs, lens[0]).numpy()
    xb = make(world, x)
    aopt = world.analysis_option(fs, api.F0_HARVEST)
    fft, dims = aopt.cheaptrick.fft_size, 60
    assert fft == 4096 and ref.number_of_aperiodicities(fs) == 5
    t, f0, fl = world.harvest(xb, fs, x_lengths=lens)
    sp = world.cheaptrick(xb, fs, t, f0, aopt.cheaptrick, x_lengths=lens, f0_lengths=fl)
    ap = world.d4c(xb, fs, t, f0, fft, x_lengths=lens, f0_lengths=fl)
    csp = world.cheaptrick_coded(xb, fs, t, f0, dims, aopt.cheaptrick, x_lengths=lens, f0_lengths=fl)
    cap = world.d4c_coded(xb, fs, t, f0, fft, x_lengths=lens, f0_lengths=fl)
    chain = world.analyze_batch(xb, fs, aopt, x_lengths=lens)
    world.synchronize()
    host = world.analyze_host(x, fs, aopt, x_lengths=lens)
    worst = {"f0": 0.0, "sp": 0.0, "ap": 0.0}
    for u in range(n_utt):
        m, xu = fl[u], x[u, :lens[u]]
        tr, fr = ref.harvest(xu, fs)
        spr = ref.cheaptrick(xu, fs, tr, fr, ref.cheaptrick_option(fs))
        apr = ref.d4c(xu, fs, tr, fr, fft)
        assert len(tr) == m and (fr > 0).sum() > 10
        for name, (tt, ff, ss, aa) in (("stages", (t, f0, sp, ap)), ("analyze_batch", chain[:4]),
                                       ("analyze_host", host[:4])):
            g = to_np(ff)[u, :m]
            assert np.array_equal(to_np(tt)[u, :m], tr), f"{name} time axis fs {fs} utt {u}"
            assert not ((g > 0) != (fr > 0)).any(), f"{name} V/UV flip fs {fs} utt {u}"
            assert_close(g, fr, f"{name} f0 fs {fs} utt {u}")
            assert_close(to_np(ss)[u, :m], spr, f"{name} spectrogram fs {fs} utt {u}")
            assert_close(to_np(aa)[u, :m], apr, f"{name} aperiodicity fs {fs} utt {u}")
            worst["f0"] = max(worst["f0"], rel_err(g, fr).max())
            worst["sp"] = max(worst["sp"], rel_err(to_np(ss)[u, :m], spr).max())
            worst["ap"] = max(worst["ap"], rel_err(to_np(aa)[u, :m], apr).max())
        c_sp = ref.code_spectral_envelope(spr, fs, fft, dims)
        c_ap = ref.code_aperiodicity(apr, fs, fft)
        assert_close_signed(to_np(csp)[u, :m], c_sp, f"coded CheapTrick fs {fs} utt {u}")
        assert_close_signed(to_np(cap)[u, :m], c_ap, f"coded D4C fs {fs} utt {u}")
        # the codec on the reference's rows
        got = (world.code_spectral_envelope(make(world, spr[None]), fs, fft, dims),
               world.code_aperiodicity(make(world, apr[None]), fs, fft),
               world.decode_spectral_envelope(make(world, c_sp[None]), fs, fft, dims),
               world.decode_aperiodicity(make(world, c_ap[None]), fs, fft))
        world.synchronize()
        assert_close_signed(to_np(got[0])[0], c_sp, f"CodeSpectralEnvelope fs {fs}")
        assert_close_signed(to_np(got[1])[0], c_ap, f"CodeAperiodicity fs {fs}")
        assert_close(to_np(got[2])[0], ref.decode_spectral_envelope(c_sp, fs, fft, dims), f"DecodeSpectralEnvelope fs {fs}")
        assert_close(to_np(got[3])[0], ref.decode_aperiodicity(c_ap, fs, fft), f"DecodeAperiodicity fs {fs}")
    return worst


def high_rate_rejections(world, fs):
    """(name, call) pairs that must fail with WORLD_B200_EINVAL at fs > 48 kHz: StoneMask has no twiddles for it,
    so neither has the DIO chain of analyze_batch."""
    from synth import synth_batch
    from world_b200 import api
    n = fs // 5
    x = make(world, synth_batch([9], fs, n).numpy())
    L = world.frames(fs, n)
    t = make(world, (np.arange(L) * 0.005)[None])
    f = make(world, np.full((1, L), 150.0))
    return [(f"StoneMask fs={fs}", lambda: world.stonemask(x, fs, t, f)),
            (f"analyze_batch F0_DIO_STONEMASK fs={fs}",
             lambda: world.analyze_batch(x, fs, world.analysis_option(fs, api.F0_DIO_STONEMASK)))]


# ---------------------------------------------------------------- 4. Synthesis
FIXED_SYNTHESIS_CASES = [
    # (fs, frame period, seconds, f0 in Hz: a constant or (start, end) of a linear ramp)
    (16000, 5.0, 2.0, 1250.0),          # 2500 pulses: beyond 1200 pulses / s + 64
    (16000, 5.0, 0.5, 1350.0),
    (16000, 2.5, 1.0, (100.0, 2400.0)),
    (16000, 5.0, 1.0, (800.0, 2400.0)),  # about 1,600 pulses, unevenly spaced: beyond the cap of 1,264
    (44100, 10.0, 0.8, (2400.0, 900.0)),  # about 1,320 pulses against a cap of 1,024
    (22050, 10.0, 1.0, 2000.0),
    (48000, 5.0, 0.6, (2200.0, 80.0)),
]


def _synthesis_params(ref, rng, fs, fp, n):
    """f0 / envelope / aperiodicity of a synthetic utterance from the reference's own DIO + StoneMask + CheapTrick +
    D4C at frame period fp."""
    from synth import synth_batch
    x = synth_batch([int(rng.integers(1, 1 << 30))], fs, n).numpy()[0]
    o = ref.dio_option(); o.frame_period = fp
    t, f0 = ref.dio(x, fs, o)
    f0 = ref.stonemask(x, fs, t, f0)
    co = ref.cheaptrick_option(fs)
    return f0, ref.cheaptrick(x, fs, t, f0, co), ref.d4c(x, fs, t, f0, co.fft_size), co.fft_size


def check_synthesis_sweep(world, ref, n_random, seed, max_utts):
    """Seeded batches of 1..max_utts utterances, one call each, with f0_lengths / y_lengths: rates 16 to 48 kHz
    (fft 1024 / 2048), frame periods 2.5 / 5 / 10 ms, y_length shorter and longer than the parameters, pitch shifts
    x0.5..x2, unvoiced holes, f0 below the synthesis floor, and the fixed cases above (constant and ramped f0 up to
    2.4 kHz)."""
    rng = np.random.default_rng(seed)
    cases = []
    for fs, fp, secs, spec in FIXED_SYNTHESIS_CASES:
        cases.append((fs, fp, [(secs, spec)]))
    for _ in range(n_random):
        fs = int(rng.choice([16000, 22050, 44100, 48000]))
        fp = float(rng.choice([2.5, 5.0, 10.0]))
        cases.append((fs, fp, [(float(rng.uniform(0.15, 0.6)), None) for _ in range(int(rng.integers(1, max_utts + 1)))]))
    worst = 0.0
    for case, (fs, fp, utts) in enumerate(cases):
        rows = []
        for secs, spec in utts:
            n = int(secs * fs)
            f0, sp, ap, fft = _synthesis_params(ref, rng, fs, fp, n)
            if spec is not None:
                f0 = (np.full(len(f0), spec) if np.isscalar(spec) else np.linspace(spec[0], spec[1], len(f0)))
            else:
                kind = int(rng.integers(0, 4))
                if kind == 1:
                    f0 = f0 * rng.uniform(0.5, 2.0)                          # pitch shift
                elif kind == 2:
                    f0[rng.uniform(size=len(f0)) < 0.3] = 0.0                # unvoiced holes
                elif kind == 3:
                    f0[::7] = fs / fft * 0.5                                 # below the synthesis floor
            y_len = int(n * rng.uniform(0.6, 1.3)) if spec is None else n
            rows.append((f0, sp, ap, y_len))
        fft = 1024 if fs < 44100 else 2048
        bins = fft // 2 + 1
        U, L, Y = len(rows), max(len(r[0]) for r in rows), max(r[3] for r in rows)
        F = np.zeros((U, L)); S = np.ones((U, L, bins)); A = np.ones((U, L, bins))
        for u, (f0, sp, ap, _) in enumerate(rows):
            F[u, :len(f0)] = f0; S[u, :len(f0)] = sp; A[u, :len(f0)] = ap
        y = world.synthesis(make(world, F), make(world, S), make(world, A), fft, fp, fs, Y,
                            f0_lengths=[len(r[0]) for r in rows], y_lengths=[r[3] for r in rows])
        world.synchronize()                                  # a device status word is a failure too
        for u, (f0, sp, ap, y_len) in enumerate(rows):
            yr = ref.synthesis(f0, sp, ap, fft, fp, fs, y_len)
            e = np.abs(to_np(y)[u, :y_len] - yr).max() / max(np.abs(yr).max(), 1e-300)
            assert e <= 1e-9, (f"Synthesis case {case} utt {u}: fs {fs} fp {fp} f0 max {f0.max():.0f} Hz, "
                               f"{e:.2e} of the peak")
            worst = max(worst, e)
    return worst


# ---------------------------------------------------------------- the tests: emulation (CPU suite) ...
@pytest.mark.parametrize("stage", list(CHUNK_CHECKS))
def test_emu_scratch_chunks(emu, ref, stage):
    print(f"{stage}: worst {CHUNK_CHECKS[stage](emu, ref):.2e}")


@pytest.mark.parametrize("fs", [16000, 22050, 44100, 48000])
def test_emu_d4c_fast_slow_split(emu, ref, fs):
    print(f"fs {fs}: worst {check_d4c_split(emu, ref, fs):.2e}")


@pytest.mark.parametrize("fs", [88200, 96000])
def test_emu_high_rate_harvest_chain(emu, ref, fs):
    n = int(0.3 * fs)
    print(f"fs {fs}: worst {check_high_rate_chain(emu, ref, fs, [n, n - int(0.07 * fs)])}")


@pytest.mark.parametrize("fs", [88200, 96000])
def test_emu_high_rate_dio_chain_rejected(emu, fs):
    from world_b200.api import WorldError
    for name, call in high_rate_rejections(emu, fs):
        with pytest.raises(WorldError, match="error 3"):
            call()
    emu.synchronize()


def test_emu_synthesis_sweep(emu, ref):
    print(f"worst {check_synthesis_sweep(emu, ref, n_random=6, seed=11, max_utts=2):.2e} of the peak")


# ---------------------------------------------------------------- ... and the CUDA library
@pytest.mark.gpu
@pytest.mark.parametrize("stage", list(CHUNK_CHECKS))
def test_gpu_scratch_chunks(gpu_world, ref, stage):
    print(f"{stage}: worst {CHUNK_CHECKS[stage](gpu_world, ref):.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("fs", [16000, 22050, 44100, 48000])
def test_gpu_d4c_fast_slow_split(gpu_world, ref, fs):
    print(f"fs {fs}: worst {check_d4c_split(gpu_world, ref, fs):.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("fs", [88200, 96000])
def test_gpu_high_rate_harvest_chain(gpu_world, ref, fs):
    n = 10 * fs
    print(f"fs {fs}: worst {check_high_rate_chain(gpu_world, ref, fs, [n, n - int(2.9 * fs)])}")


@pytest.mark.gpu
def test_gpu_synthesis_sweep(gpu_world, ref):
    print(f"worst {check_synthesis_sweep(gpu_world, ref, n_random=30, seed=12, max_utts=4):.2e} of the peak")
