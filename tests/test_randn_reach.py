"""The randn() stream past its first million draws.  CheapTrick, D4C and Synthesis consume the reference's sequential
randn() stream (matlabfunctions.cpp:237-264); the library rebuilds it in parallel (wb_rng.cu: per-frame draw counts,
a scan to offsets, and rng_fill_kernel, whose threads jump to their 128-draw chunk with one GF(2) table per set bit of
the chunk index).  These tests pin that machinery where stage parity on speech cannot see it:

  * known answers of the production generator (world_b200_randn_window) against an independent restatement of the
    stream (randn_ref.py) across every chunk-index bit, mid-chunk and mid-warp-tile window edges and the last draws
    the tables reach;
  * CheapTrick on digital silence, where every output bin is a function of the frame's draws alone, over more than
    2^24 draws per utterance;
  * D4C on a quiet voiced signal, where the 1e-6 safeguard noise decides the upper bands, past 2^22 draws with pass B
    continuing after pass A;
  * Synthesis at 48 kHz past 2^22 draws, where the noise is at full scale;
  * the reach: an utterance that would draw past 2^31 numbers is refused with WORLD_B200_EDOMAIN instead of reusing
    the stream from draw 0.

Each check runs on the host emulation (CPU suite) and on the CUDA library (-m gpu) unless marked GPU only."""
import ctypes as C

import numpy as np
import pytest

import randn_ref
from test_parity_common import assert_close, make, to_np
from test_stage_paths import SMALL_BUDGET, _with_budget

REACH = 1 << 31          # draws per utterance the library reproduces (128-draw chunks x 2^24)
FS = 48000
FFT = 2048               # CheapTrick's default at 48 kHz
BINS = FFT // 2 + 1
F0_2048 = 72000.0 / 511  # h = round(1.5 fs / f0) = 511: 2h + 1 + bins = 2048 draws per frame
TIES = (128.0, 384.0, 640.0, 1152.0)   # 1.5 fs / f0 = 562.5, 187.5, 112.5, 62.5 exactly (rounded away from zero)


def _round_half_away(v):
    return np.floor(np.abs(v) + 0.5) * np.sign(v)


def _hook(world, first, n):
    out = make(world, np.zeros(n, dtype=np.uint32), dtype=np.uint32)
    world.randn_window(first, n, out)
    world.synchronize()
    return to_np(out)


# ---------------------------------------------------------------- 1. the generator through the window hook
def _windows():
    """(first, n): every chunk-index bit's boundary 128 * 2^k, straddled from a mid-chunk start; windows that start and
    end inside a chunk and inside a 4096-draw warp tile, or span several tiles; the last draws below the reach"""
    w = [(128 * (1 << k) - 37, 75) for k in range(24)]
    w += [(0, 1), (5, 3), (127, 2), (4095, 2), (4000, 200), (4096 * 3 + 77, 4096 * 2 + 1000), (1000003, 5000),
          (123456789, 9000), ((1 << 24) * 128 // 2 + 4096 * 5 - 1, 33), (REACH - 4096 - 300, 4396), (REACH - 1, 1)]
    return w


def check_windows(world):
    for first, n in _windows():
        got = _hook(world, first, n)
        want = randn_ref.window(first, n)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"draws [{first}, {first + n}): first mismatch at draw {first + bad[0]}"


def check_window_limits(world):
    from world_b200.api import WorldError
    out = make(world, np.zeros(8, dtype=np.uint32), dtype=np.uint32)
    for first, n in ((REACH - 4, 5), (REACH, 1), (1 << 40, 1)):
        with pytest.raises(WorldError, match="error 3"):
            world.randn_window(first, n, out)
    world.randn_window(REACH, 0, out)          # empty window at the reach: nothing to do
    world.synchronize()


def test_reference_stream_anchor(ref, golden):
    """randn_ref against the reference's own randn() called in sequence (10^5 draws) and the golden known answers."""
    from test_helpers import bind
    L = bind(ref.lib)
    st = (C.c_uint32 * 4)()
    L.randn_reseed(st)
    seq = np.array([L.randn(st) for _ in range(100000)])
    mine = randn_ref.values(randn_ref.window(0, 100000))
    assert np.array_equal(mine, seq)
    assert np.array_equal(mine[:32], golden["randn_first32"])
    assert np.array_equal(randn_ref.values(randn_ref.window(1000000, 8)), golden["randn_at_1e6"])
    # the jump agrees with stepping: a window from a jumped state continues the sequential stream
    assert np.array_equal(randn_ref.window(99990, 10), randn_ref.window(0, 100000)[99990:])


# ---------------------------------------------------------------- 2. CheapTrick on digital silence
def ct_counts(f0):
    """draws per frame of CheapTrick at 48 kHz, fft 2048 (cheaptrick.cpp:210-222): 2h + 1 + bins"""
    floor = 3.0 * FS / (FFT - 3.0)
    f = np.where(f0 <= floor, 500.0, f0)
    return (2 * _round_half_away(1.5 * FS / f) + 1 + BINS).astype(np.int64)


def _silence_contours(rng, frames):
    """Mostly 2048-draw frames (the offset advances 16 chunks a frame), and among them unvoiced frames (500 Hz),
    f0 below CheapTrick's floor, rounding ties of 1.5 fs / f0 (odd and even h) and random f0."""
    rows = []
    for n in frames:
        f = np.full(n, F0_2048)
        kind = rng.integers(0, 20, size=n)
        f[kind == 0] = 0.0
        f[kind == 1] = 50.0
        f[kind == 2] = rng.choice(TIES, size=int((kind == 2).sum()))
        f[kind == 3] = rng.uniform(71.0, 800.0, size=int((kind == 3).sum()))
        rows.append(f)
    return rows


def check_cheaptrick_silence(world, ref):
    rng = np.random.default_rng(5)
    frames = [9000, 2500, 4100]
    lens = [4800, 3100, 4000]
    rows = _silence_contours(rng, frames)
    assert ct_counts(rows[0]).sum() > (1 << 24) + 4096      # utterance 0 crosses every chunk-index bit up to 2^24 draws
    U, L = len(frames), max(frames)
    x = np.zeros((U, max(lens)))
    t = np.zeros((U, L)); f = np.zeros((U, L))
    for u, n in enumerate(frames):
        t[u, :n] = rng.integers(0, lens[u], size=n) / FS      # sparse, repeated positions: silence everywhere
        f[u, :n] = rows[u]
    xb, tb, fb = make(world, x), make(world, t), make(world, f)
    small = _with_budget(world, SMALL_BUDGET)                 # one utterance per pass (u0 > 0)
    try:
        outs = []
        for w in (world, small):
            outs.append(w.cheaptrick(xb, FS, tb, fb, w.cheaptrick_option(FS), x_lengths=lens, f0_lengths=frames))
            w.synchronize()
    finally:
        small.close()
    for u, n in enumerate(frames):
        want = ref.cheaptrick(x[u, :lens[u]], FS, t[u, :n], f[u, :n])
        for name, sp in zip(("one pass", "64 MB budget"), outs):
            assert_close(to_np(sp)[u, :n], want, f"CheapTrick on silence utt {u} ({name})")


# ---------------------------------------------------------------- 3. D4C on a quiet voiced signal
def _quiet_voiced(f0_frames, n, amp, gaps):
    """Harmonics below 2 kHz along the 5 ms f0 contour at amplitude amp (the 1e-6 safeguard noise decides the bands
    above), silent where f0 is 0 and inside the sample ranges `gaps` (LoveTrain rejects those frames)."""
    tf = np.arange(len(f0_frames)) * 0.005
    fi = np.interp(np.arange(n) / FS, tf, np.where(f0_frames > 0, f0_frames, 0.0))
    phase = np.cumsum(2 * np.pi * fi / FS)
    x = np.zeros(n)
    for k in range(1, 60):
        live = (k * fi < 2000.0) & (fi > 0)
        x += live * np.sin(k * phase) / k
    for a, b in gaps:
        x[a:b] = 0.0
    return amp * x


def d4c_counts(f0):
    a = np.where(f0 > 0, 2 * _round_half_away(1.5 * FS / np.maximum(f0, 40.0)) + 1, 0).astype(np.int64)
    b = 3 * (2 * _round_half_away(2.0 * FS / np.maximum(f0, 47.0)) + 1).astype(np.int64)
    return a, b


def check_d4c_quiet(world, ref):
    # f0 around D4C's clamps (40 Hz in pass A, 47 Hz in pass B) and on both sides of the fast / slow body split
    # (75 Hz at 48 kHz); utterance 1 is shorter with a different mix, so each utterance has its own pass-B base
    base = np.concatenate([np.full(60, 35.0), np.full(60, 40.0), np.linspace(40.0, 47.0, 80), np.full(60, 47.0),
                           np.linspace(47.0, 75.0, 140), np.linspace(75.0, 130.0, 100), np.full(60, 43.0)])
    f0s = [base.copy(), np.concatenate([base[::-1][:300], np.full(40, 90.0)])]
    f0s[0][::23] = 0.0
    f0s[1][7::31] = 0.0
    frames = [len(c) for c in f0s]
    lens = [int((m - 1) * 0.005 * FS) + FS // 10 for m in frames]
    gaps = [[(int(1.3 * FS), int(1.6 * FS)), (int(2.6 * FS), int(2.75 * FS))], [(int(0.5 * FS), int(0.8 * FS))]]
    amps = [5e-5, 2e-5]
    U, L = 2, max(frames)
    x = np.zeros((U, max(lens))); t = np.zeros((U, L)); f = np.zeros((U, L))
    for u in range(U):
        x[u, :lens[u]] = _quiet_voiced(f0s[u], lens[u], amps[u], gaps[u])
        t[u, :frames[u]] = np.arange(frames[u]) * 0.005
        f[u, :frames[u]] = f0s[u]
    xb, tb, fb = make(world, x), make(world, t), make(world, f)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs = []
        for w in (world, small):
            outs.append(w.d4c(xb, FS, tb, fb, FFT, x_lengths=lens, f0_lengths=frames))
            w.synchronize()
    finally:
        small.close()
    for u in range(U):
        m = frames[u]
        want = ref.d4c(x[u, :lens[u]], FS, t[u, :m], f[u, :m], FFT)
        selected = ~np.all(want == 1.0 - 1e-12, axis=1)
        rejected_voiced = (~selected) & (f0s[u] > 0)
        assert selected.sum() > 100 and rejected_voiced.sum() > 10, (selected.sum(), rejected_voiced.sum())
        ca, cb = d4c_counts(f0s[u])
        if u == 0:
            assert ca.sum() + cb[selected].sum() > (1 << 22)   # pass-B offsets reach past 2^22
        for name, ap in zip(("one pass", "64 MB budget"), outs):
            assert_close(to_np(ap)[u, :m], want, f"D4C on a quiet signal utt {u} ({name})")


# ---------------------------------------------------------------- 4. Synthesis past 2^22 draws
def check_synthesis_long(world, ref):
    """48 kHz, fft 2048, 10 ms frames; utterance 0 lasts 90 s (about 4.3 M draws: one per sample between pulses),
    utterance 1 is shorter.  Aperiodicity near 1 above 2 kHz keeps the noise at full scale."""
    rng = np.random.default_rng(23)
    fp = 10.0
    secs = [90.0, 31.0]
    ylens = [int(s * FS) for s in secs]
    flens = [int(s * 1000 / fp) + 1 for s in secs]
    U, L = 2, max(flens)
    k = np.arange(BINS) / BINS
    F = np.zeros((U, L)); S = np.ones((U, L, BINS)); A = np.ones((U, L, BINS))
    for u in range(U):
        m = flens[u]
        f = rng.uniform(80.0, 260.0) * (1 + 0.3 * np.sin(np.arange(m) / 40.0))
        f[rng.uniform(size=m) < 0.2] = 0.0
        F[u, :m] = f
        S[u, :m] = np.exp(-5.0 * k[None, :] + 0.3 * rng.normal(size=(m, 1))) * 1e-3
        A[u, :m] = np.clip(0.05 + k[None, :] * 4 + 0.05 * rng.uniform(size=(m, BINS)), 1e-3, 1 - 1e-12)
    y = world.synthesis(make(world, F), make(world, S), make(world, A), FFT, fp, FS, max(ylens),
                        f0_lengths=flens, y_lengths=ylens)
    world.synchronize()
    for u in range(U):
        yr = ref.synthesis(F[u, :flens[u]], S[u, :flens[u]], A[u, :flens[u]], FFT, fp, FS, ylens[u])
        e = np.abs(to_np(y)[u, :ylens[u]] - yr).max() / np.abs(yr).max()
        assert e <= 1e-9, f"Synthesis utt {u} ({secs[u]} s at 48 kHz): {e:.2e} of the peak"


# ---------------------------------------------------------------- 5. the reach (GPU only)
def check_reach(world, frames):
    """Coded CheapTrick on silence with `frames` frames at one position, each drawing 2048 numbers: the draws of the
    utterance total 2048 * frames.  Returns the coded rows, or raises WorldError from synchronize()."""
    fs_len = 4800
    x = make(world, np.zeros((1, fs_len)))
    t = make(world, np.full((1, frames), 0.05))
    f = make(world, np.full((1, frames), F0_2048))
    try:
        out = world.cheaptrick_coded(x, FS, t, f, 8, world.cheaptrick_option(FS))
        world.synchronize()
        return out
    finally:
        world.trim()


def _free_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


# ---------------------------------------------------------------- the tests: emulation (CPU suite) ...
def test_emu_randn_windows(emu):
    check_windows(emu)
    check_window_limits(emu)


def test_emu_cheaptrick_silence(emu, ref):
    check_cheaptrick_silence(emu, ref)


def test_emu_d4c_quiet(emu, ref):
    check_d4c_quiet(emu, ref)


def test_emu_synthesis_long(emu, ref):
    check_synthesis_long(emu, ref)


# ---------------------------------------------------------------- ... and the CUDA library
@pytest.mark.gpu
def test_gpu_randn_windows(gpu_world):
    check_windows(gpu_world)
    check_window_limits(gpu_world)


@pytest.mark.gpu
def test_gpu_cheaptrick_silence(gpu_world, ref):
    check_cheaptrick_silence(gpu_world, ref)


@pytest.mark.gpu
def test_gpu_d4c_quiet(gpu_world, ref):
    check_d4c_quiet(gpu_world, ref)


@pytest.mark.gpu
def test_gpu_synthesis_long(gpu_world, ref):
    check_synthesis_long(gpu_world, ref)


@pytest.mark.gpu
def test_gpu_randn_reach(gpu_world):
    """2^20 frames of 2048 draws end exactly at the reach and succeed; two more frames would need draws
    [2^31, 2^31 + 4096), which the library does not reproduce (it used to restart the stream there, so row 2^20
    equalled row 0): the call reports WORLD_B200_EDOMAIN."""
    from world_b200.api import WorldError
    n = REACH // 2048
    need = n * 3073 * 4 + (64 << 20) * 4       # the draw scratch of the longest run, and room for its rows
    if _free_bytes() < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory; the device has "
                    f"{_free_bytes() / 2**30:.1f} GiB")
    got = _hook(gpu_world, REACH - 2048, 2048)
    assert np.array_equal(got, randn_ref.window(REACH - 2048, 2048))
    rows = to_np(check_reach(gpu_world, n))[0]
    assert not np.array_equal(rows[n - 1], rows[0]) and not np.array_equal(rows[n // 2], rows[0])
    del rows
    with pytest.raises(WorldError, match="error 4.*2\\^31 draws"):
        check_reach(gpu_world, n + 2)
