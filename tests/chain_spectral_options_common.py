"""Checks of the full-row analysis chains with one CheapTrick / D4C option per utterance
(world_b200_analyze_batch_spectral_options, world_b200_analyze_host_spectral_options and the all-gather variants); the
same assertions run against the host emulation (CPU) and the CUDA library (-m gpu)."""
import os

import numpy as np
import pytest

import dio_ranges_common as dr
import f0_ranges_common as hr
import test_parity_common as pc
from refworld import rel_err
from spectral_options_common import FLOORS, SMALL_BUDGET, ct_options, mixed_batch
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST, WorldError

# one D4C threshold per speaker of FLOORS, so that the D4C options differ between utterances as well
THRESHOLDS = [0.85, 0.6, 0.7, 0.5]


class Case:
    """A mixed batch whose sizes are interleaved (speaker k = (3u + 1) % 4 of FLOORS) and its per-utterance options:
    CheapTrick's fft_size from the speaker's floor, D4C's threshold from THRESHOLDS and, with f0_options, the chain's F0
    method searching from that floor too."""

    def __init__(self, world, fs, n_samples, n_utts, seed=11, method="harvest", f0_options=True):
        self.fs, self.method = fs, method
        self.x, _, _, self.lens, _ = mixed_batch(fs, n_samples, n_utts, seed)
        self.speaker = [(3 * u + 1) % len(FLOORS) for u in range(n_utts)]
        floors = [FLOORS[k] for k in self.speaker]
        self.ao = world.analysis_option(fs, F0_HARVEST if method == "harvest" else F0_DIO_STONEMASK)
        d4 = []
        for k in self.speaker:
            d = world.d4c_option()
            d.threshold = THRESHOLDS[k]
            d4.append(d)
        self.kw = {"cheaptrick_options": ct_options(world, fs, floors), "d4c_options": d4}
        if f0_options and method == "harvest":
            self.kw["harvest_options"] = hr.options([(lo, 800.0) for lo in floors])
        elif f0_options:
            self.kw["dio_options"] = dr.options([(lo, 800.0, 2.0, 0.1) for lo in floors])
        self.sizes = [o.fft_size for o in self.kw["cheaptrick_options"]]
        self.frames = [world.frames(fs, n, 5.0) for n in self.lens]
        self.width = max(self.sizes) // 2 + 1
        assert len(set(self.sizes)) > 1

    def run(self, world, **kw):
        """analyze_batch with the case's options (kw on top) -> numpy (t, f0, sp, ap)."""
        got = world.analyze_batch(pc.make(world, self.x), self.fs, self.ao, x_lengths=self.lens, **self.kw, **kw)
        world.synchronize()
        return [pc.to_np(a) for a in got[:4]]

    def run_host(self, world, **kw):
        got = world.analyze_host(np.ascontiguousarray(self.x), self.fs, self.ao, x_lengths=self.lens, **self.kw, **kw)
        return list(got[:4])

    def assert_rows_equal(self, got, want, what):
        """The computed part of every utterance's rows: frames [0, F), values [0, fft_size / 2 + 1)."""
        for u, (F, fft) in enumerate(zip(self.frames, self.sizes)):
            bins = fft // 2 + 1
            for name, g, w in zip(("time axis", "f0"), got[:2], want[:2]):
                assert np.array_equal(g[u, :F], w[u, :F]), f"{what}: {name}, utterance {u}"
            for name, g, w in zip(("spectrogram", "aperiodicity"), got[2:], want[2:]):
                assert np.array_equal(g[u, :F, :bins], w[u, :F, :bins]), f"{what}: {name}, utterance {u} fft {fft}"


class _Env:
    """Environment variables set for the duration of a with block."""

    def __init__(self, **values):
        self.values, self.saved = values, {}

    def __enter__(self):
        for k, v in self.values.items():
            self.saved[k] = os.environ.get(k)
            os.environ[k] = str(v)

    def __exit__(self, *exc):
        for k, v in self.saved.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def check_groups(world, fs, n_samples, n_utts, method="harvest", f0_options=True):
    """Each row of the mixed call equals, bit for bit, analyze_batch with one option on that utterance's speaker
    group alone (its size, threshold and F0 range); f0 and the time axis too."""
    c = Case(world, fs, n_samples, n_utts, method=method, f0_options=f0_options)
    got = c.run(world)
    assert got[2].shape[-1] == got[3].shape[-1] == c.width
    for k in sorted(set(c.speaker)):
        idx = [u for u in range(n_utts) if c.speaker[u] == k]
        ao = world.analysis_option(fs, c.ao.f0_method)
        ao.cheaptrick, ao.d4c = c.kw["cheaptrick_options"][idx[0]], c.kw["d4c_options"][idx[0]]
        f0kw = {name: [v[u] for u in idx] for name, v in c.kw.items() if name in ("harvest_options", "dio_options")}
        want = world.analyze_batch(pc.make(world, c.x[idx]), fs, ao, x_lengths=[c.lens[u] for u in idx], **f0kw)
        world.synchronize()
        want = [pc.to_np(a) for a in want[:4]]
        bins = c.sizes[idx[0]] // 2 + 1
        assert want[2].shape[-1] == bins
        for j, u in enumerate(idx):
            F = c.frames[u]
            for name, g, w in zip(("time axis", "f0"), got[:2], want[:2]):
                assert np.array_equal(g[u, :F], w[j, :F]), f"{name}, utterance {u}"
            for name, g, w in zip(("spectrogram", "aperiodicity"), got[2:], want[2:]):
                assert np.array_equal(g[u, :F, :bins], w[j, :F]), f"{name}, utterance {u} fft {c.sizes[u]}"
    assert (got[1] > 0).sum() > 20


def check_layout(world, fs, n_samples, n_utts=4):
    """A row_stride 3 wider than needed: on device arrays every value past an utterance's fft_size / 2 + 1 and every
    frame past its count keeps its NaN sentinel; the host chain gives 0 there and the device call's values elsewhere."""
    c = Case(world, fs, n_samples, n_utts, seed=12)
    L, W = max(c.frames), c.width + 3
    outs = {name: pc.make(world, np.full(shape, np.nan)) for name, shape in
            (("time_axis", (n_utts, L)), ("f0", (n_utts, L)), ("spectrogram", (n_utts, L, W)),
             ("aperiodicity", (n_utts, L, W)))}
    dev = c.run(world, **outs)
    # one utterance per sub-chunk, so that utterance 0 (all frames) has a sub-chunk of its own; the first call leaves
    # its rows in the pipeline's pooled buffers, where the second call's pads lie
    with _Env(WB_HOST_SUB=1):
        c.run_host(world)
        host = c.run_host(world, spectrogram=np.full((n_utts, L, W), np.nan),
                          aperiodicity=np.full((n_utts, L, W), np.nan))
    assert c.frames[0] == L
    c.assert_rows_equal(host, dev, "host chain")
    for u, (F, fft) in enumerate(zip(c.frames, c.sizes)):
        bins = fft // 2 + 1
        for name, d, h in zip(("spectrogram", "aperiodicity"), dev[2:], host[2:]):
            assert np.isfinite(d[u, :F, :bins]).all(), f"{name}, utterance {u}"
            assert np.isnan(d[u, :F, bins:]).all() and np.isnan(d[u, F:]).all(), f"device {name} pad, utterance {u}"
            assert not h[u, :F, bins:].any() and not h[u, F:].any(), f"host {name} pad, utterance {u}"


def check_identity(world, fs, n_samples, n_utts=5, method="harvest"):
    """Equal options (the default, and a non-default q1 / threshold) with row_stride = fft_size / 2 + 1: exactly the
    arrays of analyze_batch with that one option, and of analyze_host."""
    c = Case(world, fs, n_samples, n_utts, seed=13, method=method, f0_options=False)
    xb = pc.make(world, c.x)
    for q1, thr in ((None, None), (-0.3, 0.5)):
        ao = world.analysis_option(fs, c.ao.f0_method)
        if q1 is not None:
            ao.cheaptrick.q1, ao.d4c.threshold = q1, thr
        kw = dict(x_lengths=c.lens)
        same = dict(cheaptrick_options=[ao.cheaptrick] * n_utts, d4c_options=[ao.d4c] * n_utts)
        one = world.analyze_batch(xb, fs, ao, **kw)
        got = world.analyze_batch(xb, fs, ao, **kw, **same)
        world.synchronize()
        assert got[2].shape[-1] == ao.cheaptrick.fft_size // 2 + 1
        for a, b in zip(one[:4], got[:4]):
            assert np.array_equal(pc.to_np(a), pc.to_np(b)), f"device chain, q1/threshold {q1}/{thr}"
        x = np.ascontiguousarray(c.x)
        one_h = world.analyze_host(x, fs, ao, **kw)
        got_h = world.analyze_host(x, fs, ao, **kw, **same)
        for a, b in zip(one_h[:4], got_h[:4]):
            assert np.array_equal(a, b), f"host chain, q1/threshold {q1}/{thr}"


def check_vs_ref(world, ref, fs, n_samples, n_utts=4, method="harvest"):
    """Each row within the reference's tolerance of its own chain at that utterance's options: Harvest or Dio +
    StoneMask at the utterance's F0 range, then CheapTrick and D4C at its size and threshold."""
    c = Case(world, fs, n_samples, n_utts, seed=14, method=method)
    t, f0, sp, ap = c.run(world)
    for u in range(n_utts):
        k, F, fft = c.speaker[u], c.frames[u], c.sizes[u]
        xu = np.ascontiguousarray(c.x[u, :c.lens[u]])
        if method == "harvest":
            ro = ref.harvest_option()
            ro.f0_floor, ro.f0_ceil = FLOORS[k], 800.0
            tr, fr = ref.harvest(xu, fs, ro)
        else:
            tr, fr = ref.dio(xu, fs, dr.ref_option(ref, (FLOORS[k], 800.0, 2.0, 0.1)))
            fr = ref.stonemask(xu, fs, tr, fr)
        co = ref.cheaptrick_option(fs)
        co.f0_floor, co.fft_size = FLOORS[k], fft
        do = ref.d4c_option()
        do.threshold = THRESHOLDS[k]
        spr = ref.cheaptrick(xu, fs, tr, fr, co)
        apr = ref.d4c(xu, fs, tr, fr, fft, do)
        assert len(fr) == F
        assert np.array_equal(t[u, :F], tr), f"time axis, utterance {u}"
        assert not ((f0[u, :F] > 0) != (fr > 0)).any(), f"V/UV flip, utterance {u}"
        assert rel_err(f0[u, :F], fr).max() <= pc.TOL, f"f0, utterance {u}"
        pc.assert_close(sp[u, :F, :fft // 2 + 1], spr, f"spectrogram fs={fs} utt {u} fft {fft}")
        pc.assert_close(ap[u, :F, :fft // 2 + 1], apr, f"aperiodicity fs={fs} utt {u} fft {fft}")
    assert (f0 > 0).sum() > 20


def check_slices_and_chunks(world, fs, n_samples, n_utts):
    """The device rows are identical whatever the lane slices (1, 2 or 5); the host chain gives the same rows with
    the smallest scratch budget and chunks of four / sub-chunks of two utterances, which cut the size groups."""
    from world_b200.api import World
    c = Case(world, fs, n_samples, n_utts, seed=15)
    runs = []
    for s in (1, 2, 5):
        with _Env(WB_LANE_SLICES=s):
            runs.append(c.run(world))
    for s, r in zip((2, 5), runs[1:]):
        for a, b in zip(runs[0], r):
            assert np.array_equal(a, b), f"{s} lane slices"
    small = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    small.set_scratch_budget(SMALL_BUDGET)
    with _Env(WB_HOST_CHUNK=4, WB_HOST_SUB=2, WB_HOST_TAPER_MIN=1):
        host = c.run_host(small)
    c.assert_rows_equal(host, runs[0], "host chain in chunks")


def _raises(world, fn, pattern, utt):
    with pytest.raises(WorldError, match=r"error 3"):
        fn()
    msg = world.lib.world_b200_last_error(world._h).decode()
    assert pattern in msg and f"utterance {utt})" in msg, msg


def check_invalid(world, fs=16000):
    """Each EINVAL rule of the new calls names its first bad utterance and leaves the outputs as they were."""
    c = Case(world, fs, fs // 4, 4, seed=16)
    n, L, W = 4, max(c.frames), c.width
    xb, xh = pc.make(world, c.x), np.ascontiguousarray(c.x)
    sent = [np.full((n, L), 7.0), np.full((n, L), 7.0), np.full((n, L, W), 7.0), np.full((n, L, W), 7.0)]
    dev = [pc.make(world, a) for a in sent]
    host = [a.copy() for a in sent]
    names = ("time_axis", "f0", "spectrogram", "aperiodicity")

    def calls(kw, dev_rows=dev, host_rows=host):
        """The device chain, the host chain and the full-row all-gather (checked before its communicator)."""
        args = dict(x_lengths=c.lens, **kw)
        return (lambda: world.analyze_batch(xb, fs, c.ao, **dict(zip(names, dev_rows)), **args),
                lambda: world.analyze_host(xh, fs, c.ao, **dict(zip(names, host_rows)), **args),
                lambda: world.analyze_batch_allgather(xb, fs, c.ao, *dev_rows, **args))

    def with_option(name, u, field, value):
        """The case's options with utterance u's `name` option changed."""
        kw = {k: list(v) for k, v in c.kw.items()}
        o = type(kw[name][u]).from_buffer_copy(kw[name][u])
        setattr(o, field, value)
        kw[name][u] = o
        return kw

    rules = [(with_option("cheaptrick_options", 2, "fft_size", 1000), "power of two", 2),
             (with_option("cheaptrick_options", 1, "fft_size", 16384), "power of two", 1),
             (with_option("cheaptrick_options", 3, "q1", float("nan")), "q1", 3),
             (with_option("d4c_options", 1, "threshold", float("inf")), "threshold", 1),
             (with_option("harvest_options", 2, "f0_floor", 8.0), "", 2),
             (with_option("harvest_options", 3, "frame_period", 4.0), "frame_period", 3)]
    for kw, pattern, u in rules:
        for fn in calls(kw):
            _raises(world, fn, pattern, u)
    # a row_stride below an utterance's fft_size / 2 + 1 names the first utterance of the largest size
    narrow_dev = [dev[0], dev[1], pc.make(world, sent[2][..., :W - 1]), pc.make(world, sent[3][..., :W - 1])]
    narrow_host = [host[0], host[1], sent[2][..., :W - 1].copy(), sent[3][..., :W - 1].copy()]
    for fn in calls(c.kw, narrow_dev, narrow_host):
        _raises(world, fn, "row_stride", c.sizes.index(max(c.sizes)))
    # DIO options with the Harvest method, and a DIO chain whose options break its rules
    dio_kw = dict(c.kw)
    dio_kw.pop("harvest_options")
    dio_kw["dio_options"] = dr.options([(40.0, 800.0, 2.0, 0.1)] * n)
    with pytest.raises(WorldError, match="error 3"):
        world.analyze_batch(xb, fs, c.ao, x_lengths=c.lens, **dict(zip(names, dev)), **dio_kw)
    dio_ao = world.analysis_option(fs, F0_DIO_STONEMASK)
    dio_kw["dio_options"][2].speed = 2
    for run in (lambda: world.analyze_batch(xb, fs, dio_ao, x_lengths=c.lens, **dict(zip(names, dev)), **dio_kw),
                lambda: world.analyze_host(xh, fs, dio_ao, x_lengths=c.lens, **dict(zip(names, host)), **dio_kw)):
        _raises(world, run, "", 2)
    # number_of_dimensions against every utterance's size: the coded all-gather names the first utterance at the
    # smallest size (checked before its communicator)
    cs, ca = pc.make(world, np.full((n, L, 130), 7.0)), pc.make(world, np.full((n, L, 1), 7.0))
    _raises(world, lambda: world.analyze_coded_batch_allgather(xb, 0, fs, c.ao, min(c.sizes) // 4 + 2, dev[0], dev[1],
                                                                cs, ca, x_lengths=c.lens, **c.kw),
            "number_of_dimensions", c.sizes.index(min(c.sizes)))
    world.synchronize()
    for name, want, d, h in zip(names, sent, dev, host):
        assert np.array_equal(pc.to_np(d), want) and np.array_equal(h, want), name
    assert (pc.to_np(cs) == 7.0).all() and (pc.to_np(ca) == 7.0).all()
    for name, a in zip(names[2:], narrow_dev[2:] + narrow_host[2:]):
        assert (pc.to_np(a) == 7.0).all(), name
    # the full-row all-gather needs the full arrays' last dimension as its row_stride
    with pytest.raises(ValueError, match="row_stride"):
        world.analyze_batch_allgather(xb, fs, c.ao, dev[0], dev[1], None, None, x_lengths=c.lens, **c.kw)
    # the context keeps working
    got = c.run(world)
    assert np.isfinite(got[2][0, :c.frames[0], :c.sizes[0] // 2 + 1]).all()
