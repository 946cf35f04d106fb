"""Checks of CheapTrick and D4C with one option per utterance (world_b200_cheaptrick_batch_options,
world_b200_d4c_batch_options and their coded forms); the same assertions run against the host emulation (CPU) and the
CUDA library (-m gpu)."""
import ctypes as C

import numpy as np
import pytest

import test_parity_common as pc
from refworld import rel_err
from world_b200.api import WorldError

# per-speaker F0 floors; each utterance's voice sits above its own floor.  Utterance 0 (floor 40 Hz, f0 43-49 Hz) has
# voiced frames below the default option's CheapTrick floor at every rate (47.0 Hz at 16 kHz, 64.8 Hz at 22.05 kHz,
# 70.4 Hz at 48 kHz), which the default option analyses as if they were at 500 Hz.
FLOORS = [40.0, 55.0, 71.0, 100.0]
VOICES = [46.0, 62.0, 90.0, 140.0]
SMALL_BUDGET = 64 << 20   # the smallest scratch budget world_b200_set_scratch_budget accepts


def ct_options(world, fs, floors):
    """The reference's recipe: the option's f0_floor set to the speaker's floor, fft_size derived from it."""
    out = []
    for lo in floors:
        o = world.cheaptrick_option(fs)
        o.f0_floor = lo
        o.fft_size = world.lib.GetFFTSizeForCheapTrick(fs, C.byref(o))
        out.append(o)
    return out


def mixed_batch(fs, n_samples, n_utts, seed):
    """Harmonic voices at VOICES[u % 4] with a 3 Hz vibrato of +-5 %, silent (noise only) after 80 % of each ragged
    utterance; the f0 rows are the voices' own contours, 0 where unvoiced."""
    rng = np.random.default_rng(seed)
    lens = [n_samples - (37 * u * (fs // 100)) % (n_samples // 3) for u in range(n_utts)]
    frames = [int(1000.0 * n / fs / 5.0) + 1 for n in lens]
    L = max(frames)
    x, t, f0 = np.zeros((n_utts, n_samples)), np.zeros((n_utts, L)), np.zeros((n_utts, L))
    tt = np.arange(n_samples) / fs
    for u in range(n_utts):
        base = VOICES[u % len(VOICES)]
        contour = lambda s: base * (1.0 + 0.05 * np.sin(2 * np.pi * 3.0 * s + u))   # noqa: E731
        phase = 2 * np.pi * np.cumsum(contour(tt)) / fs
        sig = sum(0.3 / k * np.sin(k * phase) for k in range(1, 11))
        end = int(0.8 * lens[u])
        sig[end:] = 0.0
        x[u, :lens[u]] = (sig + 1e-3 * rng.normal(size=n_samples))[:lens[u]]
        tu = np.arange(frames[u]) * 0.005
        t[u, :frames[u]] = tu
        f0[u, :frames[u]] = np.where(tu * fs < end, contour(tu), 0.0)
    return x, t, f0, lens, frames


def _run(world, fs, x, t, f0, lens, frames, co, sizes, dims, out_sp=None, out_ap=None):
    xb, tb, fb = pc.make(world, x), pc.make(world, t), pc.make(world, f0)
    kw = dict(x_lengths=lens, f0_lengths=frames)
    sp = world.cheaptrick(xb, fs, tb, fb, co, out=out_sp, **kw)
    ap = world.d4c(xb, fs, tb, fb, sizes, out=out_ap, **kw)
    csp = world.cheaptrick_coded(xb, fs, tb, fb, dims, co, **kw)
    cap = world.d4c_coded(xb, fs, tb, fb, sizes, **kw)
    world.synchronize()
    return tuple(pc.to_np(a) for a in (sp, ap, csp, cap))


def check_vs_ref(world, ref, fs, n_samples, n_utts=4, dims=24, seed=1):
    """Every row of a mixed-size batch, full and coded, against the reference's CheapTrick / D4C (and its
    CodeSpectralEnvelope / CodeAperiodicity) at that utterance's own option."""
    x, t, f0, lens, frames = mixed_batch(fs, n_samples, n_utts, seed)
    floors = [FLOORS[u % len(FLOORS)] for u in range(n_utts)]
    co = ct_options(world, fs, floors)
    sizes = [o.fft_size for o in co]
    assert len(set(sizes)) > 1
    sp, ap, csp, cap = _run(world, fs, x, t, f0, lens, frames, co, sizes, dims)
    assert sp.shape[-1] == ap.shape[-1] == max(sizes) // 2 + 1
    n_ap = ref.number_of_aperiodicities(fs)
    for u in range(n_utts):
        F, bins = frames[u], sizes[u] // 2 + 1
        xu, tu, fu = x[u, :lens[u]], t[u, :F], f0[u, :F]
        ro = ref.cheaptrick_option(fs)
        ro.f0_floor, ro.fft_size = floors[u], sizes[u]
        spr = ref.cheaptrick(xu, fs, tu, fu, ro)
        apr = ref.d4c(xu, fs, tu, fu, sizes[u])
        pc.assert_close(sp[u, :F, :bins], spr, f"spectrogram fs={fs} utt {u} fft {sizes[u]}")
        pc.assert_close(ap[u, :F, :bins], apr, f"aperiodicity fs={fs} utt {u} fft {sizes[u]}")
        pc.assert_close_signed(csp[u, :F], ref.code_spectral_envelope(spr, fs, sizes[u], dims),
                               f"coded spectral envelope fs={fs} utt {u}")
        if n_ap > 0:
            pc.assert_close_signed(cap[u, :F], ref.code_aperiodicity(apr, fs, sizes[u]),
                                   f"coded aperiodicity fs={fs} utt {u}")
        assert not sp[u, :, bins:].any() and not ap[u, :, bins:].any()
    # not vacuous: utterance 0's voiced frames below the default floor are what its own option changes
    dflt = world.cheaptrick_option(fs)
    floor0 = 3.0 * fs / (dflt.fft_size - 3.0)
    low = (f0[0, :frames[0]] > 0) & (f0[0, :frames[0]] <= floor0)
    assert low.sum() > 5
    sd = pc.to_np(world.cheaptrick(pc.make(world, x[:1]), fs, pc.make(world, t[:1]), pc.make(world, f0[:1]), dflt,
                                   x_lengths=lens[:1], f0_lengths=frames[:1]))
    world.synchronize()
    r = sizes[0] // dflt.fft_size
    assert r >= 2
    # the same frequencies: bin k of the default grid is bin r * k of the utterance's own
    diff = rel_err(sp[0, :frames[0], :sizes[0] // 2 + 1:r][low], sd[0, :frames[0]][low])
    assert diff.max() > 0.1


def check_identity(world, fs, n_samples, n_utts=5, dims=24, seed=2):
    """Equal options (the default, and a non-default q1 / threshold) give the one-option calls' arrays bit for bit."""
    x, t, f0, lens, frames = mixed_batch(fs, n_samples, n_utts, seed)
    xb, tb, fb = pc.make(world, x), pc.make(world, t), pc.make(world, f0)
    kw = dict(x_lengths=lens, f0_lengths=frames)
    for q1, thr in ((None, None), (-0.3, 0.5)):
        o = world.cheaptrick_option(fs)
        d = world.d4c_option()
        if q1 is not None:
            o.q1, d.threshold = q1, thr
        fft = o.fft_size
        want = [world.cheaptrick(xb, fs, tb, fb, o, **kw), world.d4c(xb, fs, tb, fb, fft, d, **kw),
                world.cheaptrick_coded(xb, fs, tb, fb, dims, o, **kw), world.d4c_coded(xb, fs, tb, fb, fft, d, **kw)]
        got = [world.cheaptrick(xb, fs, tb, fb, [o] * n_utts, **kw),
               world.d4c(xb, fs, tb, fb, [fft] * n_utts, [d] * n_utts, **kw),
               world.cheaptrick_coded(xb, fs, tb, fb, dims, [o] * n_utts, **kw),
               world.d4c_coded(xb, fs, tb, fb, [fft] * n_utts, [d] * n_utts, **kw)]
        world.synchronize()
        for name, a, b in zip(("cheaptrick", "d4c", "cheaptrick_coded", "d4c_coded"), want, got):
            assert np.array_equal(pc.to_np(a), pc.to_np(b)), f"{name} q1/threshold {q1}/{thr}"


def check_groups(world, fs, n_samples, n_utts, dims=24, seed=3, small_budget=False):
    """Each row of a mixed batch is, bit for bit, the one-option call's row for that utterance's size group run alone.
    small_budget: the mixed call runs on a context with the smallest scratch budget, so groups are cut into chunks."""
    from world_b200.api import World
    x, t, f0, lens, frames = mixed_batch(fs, n_samples, n_utts, seed)
    floors = [FLOORS[(3 * u + 1) % len(FLOORS)] for u in range(n_utts)]   # interleaved sizes
    co = ct_options(world, fs, floors)
    sizes = [o.fft_size for o in co]
    w = world
    if small_budget:
        w = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
        w.set_scratch_budget(SMALL_BUDGET)
    sp, ap, csp, cap = _run(w, fs, x, t, f0, lens, frames, co, sizes, dims)
    for fft in sorted(set(sizes)):
        idx = [u for u in range(n_utts) if sizes[u] == fft]
        o = co[idx[0]]
        fl = [frames[u] for u in idx]
        xg, tg, fg = pc.make(world, x[idx]), pc.make(world, t[idx]), pc.make(world, f0[idx])
        kw = dict(x_lengths=[lens[u] for u in idx], f0_lengths=fl)
        g = [world.cheaptrick(xg, fs, tg, fg, o, **kw), world.d4c(xg, fs, tg, fg, fft, **kw),
             world.cheaptrick_coded(xg, fs, tg, fg, dims, o, **kw), world.d4c_coded(xg, fs, tg, fg, fft, **kw)]
        world.synchronize()
        g = [pc.to_np(a) for a in g]
        bins = fft // 2 + 1
        for k, u in enumerate(idx):
            F = frames[u]
            assert np.array_equal(sp[u, :F, :bins], g[0][k, :F]), f"spectrogram utt {u} fft {fft}"
            assert np.array_equal(ap[u, :F, :bins], g[1][k, :F]), f"aperiodicity utt {u} fft {fft}"
            assert np.array_equal(csp[u, :F], g[2][k, :F]), f"coded spectral envelope utt {u} fft {fft}"
            assert np.array_equal(cap[u, :F], g[3][k, :F]), f"coded aperiodicity utt {u} fft {fft}"


def check_layout(world, fs, n_samples, n_utts=4, seed=4):
    """Rows wider than an utterance's bins (a caller's row_stride): the values past fft_size / 2 + 1 of each row, and
    every frame past the utterance's f0 length, keep what the caller put there."""
    x, t, f0, lens, frames = mixed_batch(fs, n_samples, n_utts, seed)
    co = ct_options(world, fs, [FLOORS[u % len(FLOORS)] for u in range(n_utts)])
    sizes = [o.fft_size for o in co]
    W = max(sizes) // 2 + 1 + 3
    pad = pc.make(world, np.full((n_utts, t.shape[1], W), np.nan))
    pad2 = pc.make(world, np.full((n_utts, t.shape[1], W), np.nan))
    sp, ap, _, _ = _run(world, fs, x, t, f0, lens, frames, co, sizes, 8, out_sp=pad, out_ap=pad2)
    for u in range(n_utts):
        F, bins = frames[u], sizes[u] // 2 + 1
        for a in (sp, ap):
            assert np.isfinite(a[u, :F, :bins]).all()
            assert np.isnan(a[u, :F, bins:]).all() and np.isnan(a[u, F:]).all()


def _raises(world, fn, pattern, utt):
    with pytest.raises(WorldError, match=r"error 3"):
        fn()
    msg = world.lib.world_b200_last_error(world._h).decode()
    assert pattern in msg and f"(utterance {utt})" in msg, msg


def check_invalid(world, fs=16000):
    """Each EINVAL rule, named for its first bad utterance, with the outputs left as they were."""
    n = 4
    x, t, f0, lens, frames = mixed_batch(fs, fs // 4, n, 5)
    xb, tb, fb = pc.make(world, x), pc.make(world, t), pc.make(world, f0)
    kw = dict(x_lengths=lens, f0_lengths=frames)
    co = ct_options(world, fs, [FLOORS[u] for u in range(n)])
    sizes = [o.fft_size for o in co]
    W = max(sizes) // 2 + 1
    sent = np.full((n, t.shape[1], W), 7.0)
    out = pc.make(world, sent)
    bad = ct_options(world, fs, FLOORS)
    bad[2].fft_size = 1000
    _raises(world, lambda: world.cheaptrick(xb, fs, tb, fb, bad, out=out, **kw), "power of two", 2)
    bad = ct_options(world, fs, FLOORS)
    bad[1].fft_size = 16384
    _raises(world, lambda: world.cheaptrick(xb, fs, tb, fb, bad, out=out, **kw), "power of two", 1)
    bad = ct_options(world, fs, FLOORS)
    bad[3].q1 = float("nan")
    _raises(world, lambda: world.cheaptrick(xb, fs, tb, fb, bad, out=out, **kw), "q1", 3)
    narrow = pc.make(world, np.full((n, t.shape[1], W - 1), 7.0))
    _raises(world, lambda: world.cheaptrick(xb, fs, tb, fb, co, out=narrow, **kw), "row_stride", sizes.index(max(sizes)))
    _raises(world, lambda: world.d4c(xb, fs, tb, fb, sizes, out=narrow, **kw), "row_stride", sizes.index(max(sizes)))
    _raises(world, lambda: world.d4c(xb, fs, tb, fb, [1024, 2, 1024, 1024], out=out, **kw), "at least 4", 1)
    dopt = [world.d4c_option() for _ in range(n)]
    dopt[2].threshold = float("inf")
    _raises(world, lambda: world.d4c(xb, fs, tb, fb, sizes, dopt, out=out, **kw), "threshold", 2)
    # 130 dimensions fit fft_size 1024 (at most 257) but not 512 (at most 129): the first utterance at 512 is named
    _raises(world, lambda: world.cheaptrick_coded(xb, fs, tb, fb, 130, co, **kw), "number_of_dimensions",
            sizes.index(min(sizes)))
    bad_len = list(frames)
    bad_len[1] = t.shape[1] + 1
    with pytest.raises(WorldError, match="error 3"):
        world.cheaptrick(xb, fs, tb, fb, co, out=out, x_lengths=lens, f0_lengths=bad_len)
    world.synchronize()
    assert np.array_equal(pc.to_np(out), sent) and np.array_equal(pc.to_np(narrow), sent[..., :W - 1])
    # the context keeps working
    sp = world.cheaptrick(xb, fs, tb, fb, co, **kw)
    world.synchronize()
    assert np.isfinite(pc.to_np(sp)[0, :frames[0]]).all()


def check_chain(world, fs, n_samples, n_utts, dims=24, seed=6, nbit=0):
    """world_b200_analyze_coded_batch_spectral_options: each row equals world_b200_analyze_coded_batch on that
    utterance's size group alone with the group's options, bit for bit; equal options give the one-option chain;
    world_b200_analyze_coded_host_spectral_options gives the device chain's rows."""
    from world_b200.api import HarvestOption, F0_HARVEST
    x, _, _, lens, _ = mixed_batch(fs, n_samples, n_utts, seed)
    floors = [FLOORS[(3 * u + 1) % len(FLOORS)] for u in range(n_utts)]
    co = ct_options(world, fs, floors)
    sizes = [o.fft_size for o in co]
    ho = []
    for lo in floors:
        o = HarvestOption()
        o.f0_floor, o.f0_ceil, o.frame_period = lo, 800.0, 5.0
        ho.append(o)
    ao = world.analysis_option(fs, F0_HARVEST)
    d4 = [world.d4c_option() for _ in range(n_utts)]
    xb = pc.make(world, x)
    got = world.analyze_coded_batch(xb, nbit, fs, ao, dims, x_lengths=lens, harvest_options=ho, cheaptrick_options=co,
                                    d4c_options=d4)
    world.synchronize()
    got = [pc.to_np(a) for a in got[:4]]
    fl = [int(1000.0 * n / fs / 5.0) + 1 for n in lens]
    for fft in sorted(set(sizes)):
        idx = [u for u in range(n_utts) if sizes[u] == fft]
        aog = world.analysis_option(fs, F0_HARVEST)
        aog.cheaptrick = co[idx[0]]
        want = world.analyze_coded_batch(pc.make(world, x[idx]), nbit, fs, aog, dims, x_lengths=[lens[u] for u in idx],
                                         harvest_options=[ho[u] for u in idx])
        world.synchronize()
        want = [pc.to_np(a) for a in want[:4]]
        for k, u in enumerate(idx):
            for name, g, w in zip(("time axis", "f0", "coded sp", "coded ap"), got, want):
                assert np.array_equal(g[u, :fl[u]], w[k, :fl[u]]), f"chain {name}, utterance {u} fft {fft}"
    # equal options: the one-option chain's arrays
    one = world.analyze_coded_batch(xb, nbit, fs, ao, dims, x_lengths=lens, harvest_options=ho)
    same = world.analyze_coded_batch(xb, nbit, fs, ao, dims, x_lengths=lens, harvest_options=ho,
                                     cheaptrick_options=[ao.cheaptrick] * n_utts)
    world.synchronize()
    for a, b in zip(one[:4], same[:4]):
        assert np.array_equal(pc.to_np(a), pc.to_np(b))
    # the host pipeline, in sub-chunks of two utterances (WB_HOST_SUB is read per call): the device chain's rows
    import os
    os.environ["WB_HOST_SUB"], os.environ["WB_HOST_CHUNK"] = "2", "4"
    try:
        host = world.analyze_coded_host(np.ascontiguousarray(x), nbit, fs, ao, dims, x_lengths=lens, harvest_options=ho,
                                        cheaptrick_options=co, d4c_options=d4)
    finally:
        del os.environ["WB_HOST_SUB"], os.environ["WB_HOST_CHUNK"]
    for name, g, hst in zip(("time axis", "f0", "coded sp", "coded ap"), got, host[:4]):
        for u in range(n_utts):
            assert np.array_equal(g[u, :fl[u]], hst[u, :fl[u]]), f"host chain {name}, utterance {u}"
    # a dimension count that one utterance's size cannot hold names that utterance, before anything is queued
    for run in (lambda d: world.analyze_coded_batch(xb, nbit, fs, ao, d, x_lengths=lens, cheaptrick_options=co),
                lambda d: world.analyze_coded_host(np.ascontiguousarray(x), nbit, fs, ao, d, x_lengths=lens,
                                                   cheaptrick_options=co)):
        with pytest.raises(WorldError, match="error 3"):
            run(min(sizes) // 4 + 2)
        msg = world.lib.world_b200_last_error(world._h).decode()
        assert f"(utterance {sizes.index(min(sizes))})" in msg, msg
