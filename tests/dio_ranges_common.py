"""Checks of DIO with one option per utterance (world_b200_dio_batch_options and the chains built on it) and of the
coded host chain with per-utterance options of either F0 method; the same assertions run against the host emulation
(CPU) and the CUDA library (-m gpu)."""
import os

import numpy as np
import pytest

import f0_ranges_common as hr
import test_parity_common as pc
from refworld import rel_err
from world_b200.api import DioOption, F0_DIO_STONEMASK, F0_HARVEST, WorldError

# (f0_floor, f0_ceil, channels_in_octave, allowed_range): speaker-like ranges, 40-1100 Hz and a 3-channels-per-octave
# list included, and two allowed_range values for one band list.  The default 0.1 almost never decides a frame of
# these signals; 0.005 does (check_allowed_range_decides asserts it for every batch that relies on it).
TIGHT = 0.005
RANGES = [(40.0, 1100.0, 2.0, 0.1), (71.0, 800.0, 3.0, 0.1), (100.0, 600.0, 2.0, TIGHT), (50.0, 300.0, 2.0, 0.1),
          (71.0, 800.0, 3.0, TIGHT)]


def options(ranges, speed=1, frame_period=5.0):
    out = []
    for lo, hi, ch, ar in ranges:
        o = DioOption()
        o.f0_floor, o.f0_ceil, o.channels_in_octave, o.allowed_range = lo, hi, ch, ar
        o.frame_period, o.speed = frame_period, speed
        out.append(o)
    return out


def ref_option(ref, r, speed=1):
    o = ref.dio_option()
    o.f0_floor, o.f0_ceil, o.channels_in_octave, o.allowed_range = r
    o.speed = speed
    return o


def batch(fs, n_samples, seeds, silence=None):
    """A ragged batch; silence = u puts a stretch of digital silence into utterance u."""
    x, lens = hr.ragged_batch(fs, n_samples, seeds)
    if silence is not None:
        a = lens[silence] // 3
        x[silence, a:a + lens[silence] // 4] = 0.0
    return x, lens


def check_allowed_range_decides(world, fs, x, lens, rng, speed):
    """The batch's per-utterance allowed_range is not vacuous: for at least one utterance whose allowed_range differs
    from the first utterance's, a one-option call at the first utterance's allowed_range gives a different row.  So a
    contour that used one allowed_range for the whole batch (or another utterance's) would fail the row checks."""
    ar0 = rng[0][3]
    changed = 0
    for u, r in enumerate(rng):
        if r[3] == ar0:
            continue
        xu = pc.make(world, x[u:u + 1])
        _, fa, fl = world.dio(xu, fs, options([r], speed)[0], x_lengths=lens[u:u + 1])
        _, fb, _ = world.dio(xu, fs, options([r[:3] + (ar0,)], speed)[0], x_lengths=lens[u:u + 1])
        world.synchronize()
        changed += int((pc.to_np(fa)[0, :fl[0]] != pc.to_np(fb)[0, :fl[0]]).sum())
    assert changed > 0, "no utterance of the batch depends on its own allowed_range"


def check_mixed_vs_ref(world, ref, fs, n_samples, seeds, speed=1, ranges=RANGES):
    """Every row of a mixed-option batch against the reference's Dio() at that utterance's own option."""
    x, lens = batch(fs, n_samples, seeds)
    rng = [ranges[u % len(ranges)] for u in range(len(seeds))]
    check_allowed_range_decides(world, fs, x, lens, rng, speed)
    t, f0, fl = world.dio(pc.make(world, x), fs, options(rng, speed), x_lengths=lens)
    world.synchronize()
    t, f0 = pc.to_np(t), pc.to_np(f0)
    for u in range(len(seeds)):
        tr, fr = ref.dio(x[u, :lens[u]], fs, ref_option(ref, rng[u], speed))
        got = f0[u, :fl[u]]
        assert len(tr) == fl[u]
        assert np.array_equal(t[u, :fl[u]], tr), f"time axis, utterance {u} ({rng[u]})"
        assert not ((got > 0) != (fr > 0)).any(), f"V/UV flip, utterance {u} ({rng[u]})"
        assert rel_err(got, fr).max() <= pc.TOL, f"f0, utterance {u} ({rng[u]})"
        assert (fr > 0).sum() > 10


def check_composition(world, fs, n_samples, seeds, speed=1, ranges=RANGES):
    """The mixed call gives, bit for bit, the rows of each option run alone through the one-option call (one
    utterance has a stretch of digital silence, where the ripple terms decide); an options array of identical
    defaults gives the rows of the one-option call."""
    x, lens = batch(fs, n_samples, seeds, silence=1)
    n = len(seeds)
    rng = [ranges[u % len(ranges)] for u in range(n)]
    check_allowed_range_decides(world, fs, x, lens, rng, speed)
    t, f0, fl = world.dio(pc.make(world, x), fs, options(rng, speed), x_lengths=lens)
    world.synchronize()
    t, f0 = pc.to_np(t), pc.to_np(f0)
    for r in sorted(set(rng)):
        idx = [u for u in range(n) if rng[u] == r]
        tg, fg, flg = world.dio(pc.make(world, x[idx]), fs, options([r], speed)[0], x_lengths=[lens[u] for u in idx])
        world.synchronize()
        tg, fg = pc.to_np(tg), pc.to_np(fg)
        for k, u in enumerate(idx):
            assert flg[k] == fl[u]
            assert np.array_equal(t[u, :fl[u]], tg[k, :fl[u]]), f"time axis, utterance {u} ({r})"
            assert np.array_equal(f0[u, :fl[u]], fg[k, :fl[u]]), f"f0, utterance {u} ({r}) differs from its own call"
    assert (f0[1, :fl[1]] > 0).sum() > 10
    xb = pc.make(world, x)
    default = world.dio_option()
    default.speed = speed
    t1, f1, _ = world.dio(xb, fs, default, x_lengths=lens)
    td, fd, _ = world.dio(xb, fs, [default] * n, x_lengths=lens)
    world.synchronize()
    assert np.array_equal(pc.to_np(t1), pc.to_np(td)) and np.array_equal(pc.to_np(f1), pc.to_np(fd))


SMALL_BUDGET = 64 << 20   # the smallest scratch budget world_b200_set_scratch_budget accepts


def check_scratch_chunks(world, fs=16000, seconds=6.0, seeds=(141, 142, 143, 144, 145, 146, 147)):
    """A mixed-option batch cut into scratch chunks gives the one-pass rows bit for bit: every chunk reads its own
    utterances' groups and allowed_range.  At 16 kHz a 6 s utterance needs about 20 MB of DIO scratch (complete edge
    lists of 11 bands), so the smallest budget holds three utterances per chunk and the batch takes three chunks, the
    later ones starting at utterances whose allowed_range differs from the first chunk's first utterance."""
    from world_b200.api import World
    n_samples = int(fs * seconds)
    x, lens = batch(fs, n_samples, list(seeds))
    rng = [RANGES[u % len(RANGES)] for u in range(len(seeds))]
    check_allowed_range_decides(world, fs, x, lens, rng, 1)
    small = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    small.set_scratch_budget(SMALL_BUDGET)
    xb = pc.make(world, x)
    t, f0, fl = world.dio(xb, fs, options(rng), x_lengths=lens)
    tc, fc, flc = small.dio(pc.make(small, x), fs, options(rng), x_lengths=lens)
    world.synchronize()
    small.synchronize()
    assert flc == fl
    assert np.array_equal(pc.to_np(t), pc.to_np(tc)) and np.array_equal(pc.to_np(f0), pc.to_np(fc))


def _raises(fn, pattern):
    with pytest.raises(WorldError, match=pattern):
        fn()


def check_invalid(world):
    """Options the kernels cannot serve, or that break the shared settings, are EINVAL naming the utterance; options of
    the other F0 method are EINVAL on every chain; the context keeps working."""
    fs = 16000
    x, lens = batch(fs, fs // 2, [61, 62, 63, 64])
    xb, xh = pc.make(world, x), np.ascontiguousarray(x)
    good = [(71.0, 800.0, 2.0, 0.1), (100.0, 600.0, 2.0, 0.1)] * 2
    bad = options(good)
    bad[2].f0_ceil = 40.0   # f0_ceil < f0_floor: no band
    _raises(lambda: world.dio(xb, fs, bad, x_lengths=lens), r"error 3: Dio: bad band count \(utterance 2\)")
    bad = options(good)
    bad[1].frame_period = 1.0
    _raises(lambda: world.dio(xb, fs, bad, x_lengths=lens), r"error 3: .*frame_period.*utterance 1\)")
    bad = options(good)
    bad[3].speed = 2
    _raises(lambda: world.dio(xb, fs, bad, x_lengths=lens), r"error 3: .*speed.*utterance 3\)")
    # a filter too long for shared memory: a very low floor at 48 kHz without decimation
    x48, lens48 = batch(48000, 4800, [65, 66, 67])
    bad = options([(71.0, 800.0, 2.0, 0.1), (2.0, 800.0, 2.0, 0.1), (1.0, 800.0, 2.0, 0.1)])
    _raises(lambda: world.dio(pc.make(world, x48), 48000, bad, x_lengths=lens48),
            r"error 3: Dio: filters too long for shared memory.*\(utterance 1\)")
    # options of the other F0 method, on every chain
    ao_h, ao_d = world.analysis_option(fs, F0_HARVEST), world.analysis_option(fs, F0_DIO_STONEMASK)
    dopts, hopts = options(good), hr.options([(71.0, 800.0)] * 4)
    _raises(lambda: world.analyze_batch(xb, fs, ao_h, x_lengths=lens, dio_options=dopts), "error 3")
    _raises(lambda: world.analyze_batch(xb, fs, ao_d, x_lengths=lens, harvest_options=hopts), "error 3")
    _raises(lambda: world.analyze_host(xh, fs, ao_h, x_lengths=lens, dio_options=dopts), "error 3")
    _raises(lambda: world.analyze_host(xh, fs, ao_d, x_lengths=lens, harvest_options=hopts), "error 3")
    _raises(lambda: world.analyze_coded_host(xh, 0, fs, ao_h, 20, x_lengths=lens, dio_options=dopts), "error 3")
    _raises(lambda: world.analyze_coded_host(xh, 0, fs, ao_d, 20, x_lengths=lens, harvest_options=hopts), "error 3")
    # a chain cut into chunks still names the batch's first bad utterance
    bad = options(good)
    bad[3].f0_floor = 2000.0   # above f0_ceil: no band
    env = {"WB_HOST_CHUNK": "1", "WB_HOST_SUB": "1"}
    with _env(env):
        _raises(lambda: world.analyze_host(xh, fs, ao_d, x_lengths=lens, dio_options=bad), r"utterance 3\)")
    with pytest.raises(ValueError):
        world.analyze_coded_host(xh, 0, fs, ao_d, 20, x_lengths=lens, dio_options=dopts, harvest_options=hopts)
    with pytest.raises(TypeError):   # one option for the batch belongs in the AnalysisOption, on both keywords
        world.analyze_batch(xb, fs, ao_d, x_lengths=lens, dio_options=dopts[0])
    with pytest.raises(TypeError):
        world.analyze_batch(xb, fs, ao_h, x_lengths=lens, harvest_options=hopts[0])
    t, f0, fl = world.dio(xb, fs, options(good), x_lengths=lens)
    world.synchronize()
    assert (pc.to_np(f0)[0, :fl[0]] > 0).sum() > 10


class _env:
    """Sets environment variables for the duration of a with-block and restores the previous values."""

    def __init__(self, values):
        self.values, self.saved = values, {}

    def __enter__(self):
        for k, v in self.values.items():
            self.saved[k] = os.environ.get(k)
            os.environ[k] = v

    def __exit__(self, *exc):
        for k, v in self.saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def check_coded_host(world, f0_method, fs=16000, n_samples=8000, seeds=(131, 132, 133, 134, 135), dims=24):
    """analyze_coded_host with per-utterance options of either F0 method, from int16 PCM: the f0 rows of
    analyze_host with the same options, coded rows equal to cheaptrick_coded / d4c_coded on those rows, and tiny
    chunks (the options array split between them) giving the one-chunk result."""
    x, lens = batch(fs, n_samples, list(seeds))
    pcm = np.ascontiguousarray(np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.int16))
    xd = pcm.astype(np.float64) / 32768.0
    n = len(seeds)
    ao = world.analysis_option(fs, f0_method)
    if f0_method == F0_HARVEST:
        kw = {"harvest_options": hr.options([hr.RANGES[u % len(hr.RANGES)] for u in range(n)])}
    else:
        kw = {"dio_options": options([RANGES[u % len(RANGES)] for u in range(n)])}
    t, f0, csp, cap, fl = world.analyze_coded_host(pcm, 16, fs, ao, dims, x_lengths=lens, **kw)
    th, fh, _, _, flh = world.analyze_host(np.ascontiguousarray(xd), fs, ao, x_lengths=lens, **kw)
    assert fl == flh
    assert np.array_equal(t, th) and np.array_equal(f0, fh)
    for u in range(n):
        assert (f0[u, :fl[u]] > 0).sum() > 10, f"utterance {u} unvoiced"
    xb = pc.make(world, xd)
    tb, fb = pc.make(world, t), pc.make(world, f0)
    sp_ref = pc.to_np(world.cheaptrick_coded(xb, fs, tb, fb, dims, ao.cheaptrick, x_lengths=lens, f0_lengths=fl))
    ap_ref = pc.to_np(world.d4c_coded(xb, fs, tb, fb, ao.cheaptrick.fft_size, ao.d4c, x_lengths=lens, f0_lengths=fl))
    world.synchronize()
    for u in range(n):
        assert np.array_equal(csp[u, :fl[u]], sp_ref[u, :fl[u]]), f"coded envelope, utterance {u}"
        assert np.array_equal(cap[u, :fl[u]], ap_ref[u, :fl[u]]), f"coded aperiodicity, utterance {u}"
    with _env({"WB_HOST_CHUNK": "2", "WB_HOST_SUB": "1"}):
        tc, fc, cspc, capc, _ = world.analyze_coded_host(pcm, 16, fs, ao, dims, x_lengths=lens, **kw)
    for a, b in ((t, tc), (f0, fc), (csp, cspc), (cap, capc)):
        assert np.array_equal(a, b)
