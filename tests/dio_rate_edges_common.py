"""Checks of DIO at every sampling rate, speed and F0 floor, on voices that start or end abruptly: against the
reference, against DIO's own call on the utterance alone (whatever the batch, context and scratch budget around it),
and against itself with poisoned scratch.  The same assertions run against the host emulation (CPU) and the CUDA
library (-m gpu).

The band sweep streams a tile of 2048 filtered samples at a time and finalises the frames that lie before the last
complete interval of all four event trains.  A low floor at 44.1 / 48 kHz without decimation gives bands whose trains
see only two or three events in the first tile; on a voice at full amplitude from its first sample the first frames
are then finalised from that tile alone, which is where a streaming sweep departs from interp1 on the whole list."""
import os

import numpy as np
import pytest

import dio_ranges_common as dr
import test_parity_common as pc
from refworld import rel_err
from synth import synth_batch
from world_b200.api import World, WorldError

RATES = [16000, 22050, 24000, 32000, 44100, 48000]
SPEEDS = [1, 2, 4]
FLOORS = [40.0, 45.0, 50.0, 55.0, 71.0]
CEILS = [800.0, 1100.0]
KINDS = ["onset", "end", "ramped"]
SMALL_BUDGET = dr.SMALL_BUDGET


def voice(fs, n, kind, seed, base=62.0):
    """One utterance of n samples.  "onset": a harmonic voice at `base` Hz (3 Hz vibrato of +-5 %) at full amplitude
    from sample 0, noise only after 80 %; "end": noise only for the first 20 %, then the voice up to the last sample;
    "ramped": the synth_batch voice (20 ms linear ramps), the control."""
    if kind == "ramped":
        return synth_batch([seed], fs, n).numpy()[0]
    rng = np.random.default_rng(seed)
    tt = np.arange(n) / fs
    contour = base * (1.0 + 0.05 * np.sin(2 * np.pi * 3.0 * tt + seed))
    phase = 2 * np.pi * np.cumsum(contour) / fs
    sig = sum(0.3 / k * np.sin(k * phase) for k in range(1, 11) if k * base * 1.05 < 0.45 * fs)
    if kind == "onset":
        sig[int(0.8 * n):] = 0.0
    else:
        sig[:int(0.2 * n)] = 0.0
    return sig + 1e-3 * rng.normal(size=n)


def signals(fs, kinds=KINDS, seconds=0.5, seed=11):
    """[len(kinds)][n] rows, ragged: row k is n - 37 k samples long (rows are zero past their length)."""
    n = int(fs * seconds)
    lens = [n - 37 * k for k in range(len(kinds))]
    x = np.zeros((len(kinds), n))
    for k, kind in enumerate(kinds):
        x[k, :lens[k]] = voice(fs, lens[k], kind, seed + k)
    return x, lens


def option(world, f0_floor, f0_ceil, speed, channels=2.0):
    """The option a test means: the untouched default at (71, 800), the default's fields set otherwise."""
    o = world.dio_option()
    o.speed = speed
    if (f0_floor, f0_ceil, channels) != (71.0, 800.0, 2.0):
        o.f0_floor, o.f0_ceil, o.channels_in_octave = f0_floor, f0_ceil, channels
    return o


def _assert_row(got_t, got_f, tr, fr, what):
    assert len(got_t) == len(tr), f"{what}: frame count"
    assert np.array_equal(got_t, tr), f"{what}: time axis"
    assert not ((got_f > 0) != (fr > 0)).any(), f"{what}: V/UV flip at {np.flatnonzero((got_f > 0) != (fr > 0))[:6]}"
    e = rel_err(got_f, fr)
    assert e.max() <= pc.TOL, f"{what}: f0 {e.max():.2e} at frames {np.flatnonzero(e > pc.TOL)[:6]}"


def check_vs_ref(world, ref, fs, speed, f0_ceil, floors=FLOORS, kinds=KINDS):
    """Every kind of voice at every floor against the reference's Dio(): through the one-option call (one call per
    floor over all voices) and through the per-utterance call (one call over every (voice, floor) pair)."""
    x, lens = signals(fs, kinds)
    want = {}
    for fl0 in floors:
        ro = option(ref, fl0, f0_ceil, speed)
        for k in range(len(kinds)):
            want[k, fl0] = ref.dio(np.ascontiguousarray(x[k, :lens[k]]), fs, ro)
    voiced = 0
    xb = pc.make(world, x)
    for fl0 in floors:
        t, f0, nf = world.dio(xb, fs, option(world, fl0, f0_ceil, speed), x_lengths=lens)
        world.synchronize()
        t, f0 = pc.to_np(t), pc.to_np(f0)
        for k, kind in enumerate(kinds):
            tr, fr = want[k, fl0]
            _assert_row(t[k, :nf[k]], f0[k, :nf[k]], tr, fr,
                        f"one option, {kind} voice, fs {fs}, speed {speed}, floor {fl0}, ceil {f0_ceil}")
            voiced += int((fr > 0).sum())
    pairs = [(k, fl0) for fl0 in floors for k in range(len(kinds))]
    xp = np.stack([x[k] for k, _ in pairs])
    opts = [option(world, fl0, f0_ceil, speed) for _, fl0 in pairs]
    t, f0, nf = world.dio(pc.make(world, xp), fs, opts, x_lengths=[lens[k] for k, _ in pairs])
    world.synchronize()
    t, f0 = pc.to_np(t), pc.to_np(f0)
    for u, (k, fl0) in enumerate(pairs):
        tr, fr = want[k, fl0]
        _assert_row(t[u, :nf[u]], f0[u, :nf[u]], tr, fr,
                    f"per-utterance options, {kinds[k]} voice, fs {fs}, speed {speed}, floor {fl0}, ceil {f0_ceil}")
    assert voiced > 20 * len(floors) * len(kinds), "the voices must be voiced"


def _fresh(world, budget=None):
    w = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    if budget is not None:
        w.set_scratch_budget(budget)
    return w


def _warm(world, fs):
    """DIO and Harvest calls at other floors and speeds, so that scratch and on-chip memory hold their values."""
    x = synth_batch([5, 6], fs, fs // 4).numpy()
    xb = pc.make(world, x)
    for fl0, speed in ((45.0, 2), (100.0, 1), (40.0, 4), (55.0, 1)):
        world.dio(xb, fs, option(world, fl0, 800.0, speed))
    ho = world.harvest_option()
    ho.f0_floor = 40.0
    world.harvest(xb, fs, ho)
    world.synchronize()


def check_lone(world, fs, speed, floors=(40.0, 50.0), kind="onset"):
    """The target utterance's t / f0 rows equal, bit for bit, DIO on that utterance alone in a fresh context, whatever
    surrounds it: partners with other floors and band counts (one of 1000 samples), the target first or last, a fresh
    context or one that has run DIO and Harvest before, the smallest scratch budget or the default."""
    x, lens = signals(fs, [kind, "ramped", "end"])
    target = np.ascontiguousarray(x[0, :lens[0]])
    partners = [(x[1, :lens[1]], (100.0, 600.0, 3.0)), (x[2, :1000], (71.0, 800.0, 2.0)),
                (x[2, :lens[2]], (45.0, 1100.0, 4.0))]
    lone = {}
    for fl0 in floors:
        w = _fresh(world)
        t, f0, nf = w.dio(pc.make(w, target[None]), fs, option(w, fl0, 800.0, speed))
        w.synchronize()
        lone[fl0] = pc.to_np(t)[0, :nf[0]], pc.to_np(f0)[0, :nf[0]]
        assert (lone[fl0][1] > 0).sum() > 20
    for ctx in ("fresh", "warm", "small"):
        w = _fresh(world, SMALL_BUDGET if ctx == "small" else None)
        if ctx != "fresh":
            _warm(w, fs)
        for fl0 in floors:
            mine = (target, (fl0, 800.0, 2.0))
            for order in ("first", "last", "alone"):
                rows = {"first": [mine] + partners, "last": partners + [mine], "alone": [mine]}[order]
                k = len(rows) - 1 if order == "last" else 0
                xb = np.zeros((len(rows), max(len(r) for r, _ in rows)))
                for i, (r, _) in enumerate(rows):
                    xb[i, :len(r)] = r
                opts = [option(w, lo, hi, speed, ch) for _, (lo, hi, ch) in rows]
                t, f0, nf = w.dio(pc.make(w, xb), fs, opts if len(rows) > 1 else opts[0], x_lengths=[len(r) for r, _ in rows])
                w.synchronize()
                t, f0 = pc.to_np(t)[k, :nf[k]], pc.to_np(f0)[k, :nf[k]]
                what = f"fs {fs}, speed {speed}, floor {fl0}, {order} in the batch, {ctx} context"
                assert np.array_equal(t, lone[fl0][0]), f"{what}: time axis"
                bad = np.flatnonzero(f0 != lone[fl0][1])
                assert bad.size == 0, f"{what}: f0 differs from the lone call at frames {bad[:6]}"


def _stages(world, fs, x, lens, dio_opts):
    """DIO (per-utterance options), StoneMask, Harvest, CheapTrick and D4C; every output on the host."""
    xb = pc.make(world, x)
    t, f0, nf = world.dio(xb, fs, dio_opts, x_lengths=lens)
    f0s = world.stonemask(xb, fs, t, f0, x_lengths=lens, f0_lengths=nf)
    th, fh, nh = world.harvest(xb, fs, x_lengths=lens)
    co = world.cheaptrick_option(fs)
    sp = world.cheaptrick(xb, fs, th, fh, co, x_lengths=lens, f0_lengths=nh)
    ap = world.d4c(xb, fs, th, fh, co.fft_size, x_lengths=lens, f0_lengths=nh)
    world.synchronize()
    return [pc.to_np(a).copy() for a in (t, f0, f0s, th, fh, sp, ap)]


def check_poison(world, fs=48000, poisons=("0xFF", "0x5A")):
    """WB_ARENA_POISON fills every scratch block with one byte before a stage driver gets it; 0xFF makes any stale
    double NaN.  DIO, StoneMask, Harvest, CheapTrick and D4C give bit-identical outputs under two poison bytes and
    without poison: no stage reads scratch it has not written in the same call."""
    x, lens = signals(fs, ["onset", "ramped", "end"], seconds=0.3)
    dio_opts = [option(world, lo, hi, 1, ch) for lo, hi, ch in ((50.0, 800.0, 2.0), (100.0, 600.0, 3.0),
                                                               (40.0, 1100.0, 2.0))]
    clean = _stages(world, fs, x, lens, dio_opts)
    assert (clean[1][0] > 0).sum() > 10 and (clean[4][1] > 0).sum() > 10
    names = ("dio t", "dio f0", "stonemask f0", "harvest t", "harvest f0", "cheaptrick", "d4c")
    saved = os.environ.get("WB_ARENA_POISON")
    try:
        for byte in poisons:
            os.environ["WB_ARENA_POISON"] = byte
            got = _stages(world, fs, x, lens, dio_opts)
            for name, a, b in zip(names, clean, got):
                assert a.shape == b.shape
                bad = np.argwhere(a.view(np.uint64) != b.view(np.uint64))
                assert bad.size == 0, f"{name} differs under WB_ARENA_POISON={byte} at {bad[:4].tolist()}"
        # a value that is not one byte fails the call, naming the variable, and the context keeps working
        for bad in ("", "zz", "0x100", "-1", "12abc"):
            os.environ["WB_ARENA_POISON"] = bad
            with pytest.raises(WorldError, match="WB_ARENA_POISON"):
                world.dio(pc.make(world, x), fs, dio_opts, x_lengths=lens)
        os.environ.pop("WB_ARENA_POISON")
        again = _stages(world, fs, x, lens, dio_opts)
        for name, a, b in zip(names, clean, again):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), f"{name} after a refused poison value"
    finally:
        if saved is None:
            os.environ.pop("WB_ARENA_POISON", None)
        else:
            os.environ["WB_ARENA_POISON"] = saved
