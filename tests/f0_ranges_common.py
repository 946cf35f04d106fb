"""Checks of Harvest with one F0 range per utterance (world_b200_harvest_batch_options and the chains built on it);
the same assertions run against the host emulation (CPU) and the CUDA library (-m gpu)."""
import numpy as np
import pytest

import test_parity_common as pc
from refworld import rel_err
from world_b200.api import HarvestOption, WorldError

# speaker-like ranges, 40-1100 Hz (203 channels, the reference demo's floor) included
RANGES = [(40.0, 1100.0), (71.0, 800.0), (100.0, 600.0), (50.0, 300.0), (60.0, 400.0)]


def options(ranges, frame_period=5.0):
    out = []
    for lo, hi in ranges:
        o = HarvestOption()
        o.f0_floor, o.f0_ceil, o.frame_period = lo, hi, frame_period
        out.append(o)
    return out


def ragged_batch(fs, n_samples, seeds):
    from synth import synth_batch
    x = synth_batch(seeds, fs, n_samples, device="cpu").numpy()
    lens = [n_samples - (37 * i * (fs // 100)) % (n_samples // 3) for i in range(len(seeds))]
    return x, lens


def check_mixed_vs_ref(world, ref, fs, n_samples, seeds, ranges=RANGES):
    """Every row of a mixed-range batch against the reference's Harvest at that utterance's own option."""
    x, lens = ragged_batch(fs, n_samples, seeds)
    rng = [ranges[u % len(ranges)] for u in range(len(seeds))]
    t, f0, fl = world.harvest(pc.make(world, x), fs, options(rng), x_lengths=lens)
    world.synchronize()
    t, f0 = pc.to_np(t), pc.to_np(f0)
    for u in range(len(seeds)):
        ro = ref.harvest_option()
        ro.f0_floor, ro.f0_ceil = rng[u]
        tr, fr = ref.harvest(x[u, :lens[u]], fs, ro)
        got = f0[u, :fl[u]]
        assert len(tr) == fl[u]
        assert np.array_equal(t[u, :fl[u]], tr), f"time axis, utterance {u} ({rng[u]})"
        assert not ((got > 0) != (fr > 0)).any(), f"V/UV flip, utterance {u} ({rng[u]})"
        assert rel_err(got, fr).max() <= pc.TOL, f"f0, utterance {u} ({rng[u]})"
        assert (fr > 0).sum() > 10


def check_composition(world, fs, n_samples, seeds, ranges=RANGES):
    """The mixed call gives, bit for bit, the rows of each range group run alone through the one-option call; an
    options array of identical defaults gives the rows of the one-option call."""
    x, lens = ragged_batch(fs, n_samples, seeds)
    n = len(seeds)
    rng = [ranges[u % len(ranges)] for u in range(n)]
    t, f0, fl = world.harvest(pc.make(world, x), fs, options(rng), x_lengths=lens)
    world.synchronize()
    t, f0 = pc.to_np(t), pc.to_np(f0)
    for r in sorted(set(rng)):
        idx = [u for u in range(n) if rng[u] == r]
        tg, fg, flg = world.harvest(pc.make(world, x[idx]), fs, options([r])[0], x_lengths=[lens[u] for u in idx])
        world.synchronize()
        tg, fg = pc.to_np(tg), pc.to_np(fg)
        for k, u in enumerate(idx):
            assert flg[k] == fl[u]
            assert np.array_equal(t[u, :fl[u]], tg[k, :fl[u]]), f"time axis, utterance {u} ({r})"
            assert np.array_equal(f0[u, :fl[u]], fg[k, :fl[u]]), f"f0, utterance {u} ({r}) differs from its group's call"
    xb = pc.make(world, x)
    t1, f1, _ = world.harvest(xb, fs, world.harvest_option(), x_lengths=lens)
    td, fd, _ = world.harvest(xb, fs, [world.harvest_option() for _ in range(n)], x_lengths=lens)
    world.synchronize()
    assert np.array_equal(pc.to_np(t1), pc.to_np(td)) and np.array_equal(pc.to_np(f1), pc.to_np(fd))


def check_invalid_range(world, fs):
    """A range the kernels cannot serve is EINVAL naming the first such utterance; the context keeps working."""
    x, lens = ragged_batch(fs, fs // 2, [61, 62, 63, 64])
    xb = pc.make(world, x)
    rng = [(71.0, 800.0), (100.0, 600.0), (8.0, 800.0), (4.0, 800.0)]
    with pytest.raises(WorldError, match=r"error 3: .*utterance 2\)"):
        world.harvest(xb, fs, options(rng), x_lengths=lens)
    bad_fp = options([(71.0, 800.0)] * 4)
    bad_fp[1].frame_period = 1.0
    with pytest.raises(WorldError, match=r"error 3: .*frame_period.*utterance 1\)"):
        world.harvest(xb, fs, bad_fp, x_lengths=lens)
    ao = world.analysis_option(fs, 0)   # DIO chain: per-utterance Harvest options do not apply
    with pytest.raises(WorldError, match="error 3"):
        world.analyze_batch(xb, fs, ao, x_lengths=lens, harvest_options=options([(71.0, 800.0)] * 4))
    t, f0, fl = world.harvest(xb, fs, options([(71.0, 800.0), (100.0, 600.0)] * 2), x_lengths=lens)
    world.synchronize()
    assert (pc.to_np(f0)[0, :fl[0]] > 0).sum() > 10
