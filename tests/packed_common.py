"""Checks of the packed analysis chains (world_b200_analyze_packed, world_b200_analyze_coded_packed and their host
forms): utterances back to back with n + 1 sample offsets, outputs [F] frames with F the sum of the frame counts.  Each
utterance's rows are compared bit for bit with the padded *_spectral_options chain on the same utterances; the same
assertions run against the host emulation (CPU) and the CUDA library (-m gpu)."""
import ctypes as C

import numpy as np
import pytest

import chain_spectral_options_common as cs
import test_parity_common as pc
from refworld import rel_err
from spectral_options_common import FLOORS, SMALL_BUDGET
from world_b200.api import WorldError

DIMS = 40


def pcm(x, nbit):
    """float rows -> little-endian nbit-bit PCM rows ([n, stride * nbit / 8] uint8) of 0.9 of full scale."""
    ints = np.round(x * 0.9 * (2 ** (nbit - 1) - 1)).astype("<i4")
    b = nbit // 8
    return np.ascontiguousarray(ints.view(np.uint8).reshape(*ints.shape, 4)[..., :b].reshape(ints.shape[0], -1))


class Packed:
    """A padded case of chain_spectral_options_common (interleaved FFT sizes, per-speaker D4C thresholds and, with
    f0_options, F0 ranges) and the same utterances packed; lens overrides the case's lengths."""

    def __init__(self, world, fs, n_samples, n_utts, method="harvest", f0_options=True, seed=21, lens=None,
                 spectral_options=True):
        c = cs.Case(world, fs, n_samples, max(n_utts, 4), seed=seed, method=method, f0_options=f0_options)
        if n_utts < 4:   # the case's first utterances (a case of four has two FFT sizes at every rate)
            m = n_utts
            c.x, c.lens, c.frames, c.speaker, c.sizes = c.x[:m], c.lens[:m], c.frames[:m], c.speaker[:m], c.sizes[:m]
            c.kw = {k: v[:m] for k, v in c.kw.items()}
        if lens is not None:
            c.lens = list(lens)
            c.frames = [world.frames(fs, n, 5.0) for n in c.lens]
            for u, n in enumerate(c.lens):
                c.x[u, n:] = 0.0
        if not spectral_options:
            for k in ("cheaptrick_options", "d4c_options"):
                c.kw.pop(k)
            c.sizes = [c.ao.cheaptrick.fft_size] * n_utts
            c.width = c.sizes[0] // 2 + 1
        self.c, self.fs, self.n = c, fs, n_utts
        self.xo = np.concatenate([[0], np.cumsum(c.lens)]).astype(np.int64)

    def x_packed(self, nbit=0):
        rows = self.c.x if nbit == 0 else pcm(self.c.x, nbit)
        b = 8 if nbit == 0 else nbit // 8
        flat = rows.view(np.uint8).reshape(self.n, -1) if nbit == 0 else rows
        data = np.concatenate([flat[u, :n * b] for u, n in enumerate(self.c.lens)])
        return data.view(np.float64) if nbit == 0 else data, rows

    def padded(self, world, coded=False, nbit=0, host=False):
        """The padded counterpart's (t, f0, sp, ap) as numpy [n, L, ...]."""
        c, kw = self.c, dict(x_lengths=self.c.lens, **self.c.kw)
        _, rows = self.x_packed(nbit)
        if coded and host:
            got = world.analyze_coded_host(np.ascontiguousarray(rows), nbit, self.fs, c.ao, DIMS, **kw)
        elif coded:
            got = world.analyze_coded_batch(pc.make(world, rows, rows.dtype), nbit, self.fs, c.ao, DIMS, **kw)
        elif host:
            got = world.analyze_host(np.ascontiguousarray(rows), self.fs, c.ao, **kw)
        else:
            got = world.analyze_batch(pc.make(world, rows), self.fs, c.ao, **kw)
        world.synchronize()
        return [pc.to_np(a) for a in got[:4]]

    def packed(self, world, coded=False, nbit=0, host=False, **out):
        """The packed call's (t, f0, sp, ap) as numpy and its frame offsets."""
        c = self.c
        data, _ = self.x_packed(nbit)
        if coded and host:
            got = world.analyze_coded_host_packed(data, nbit, self.xo, self.fs, c.ao, DIMS, **c.kw, **out)
        elif coded:
            got = world.analyze_coded_packed(pc.make(world, data, data.dtype), nbit, self.xo, self.fs, c.ao, DIMS,
                                             **c.kw, **out)
        elif host:
            got = world.analyze_host_packed(data, self.xo, self.fs, c.ao, **c.kw, **out)
        else:
            got = world.analyze_packed(pc.make(world, data), self.xo, self.fs, c.ao, **c.kw, **out)
        world.synchronize()
        return [pc.to_np(a) for a in got[:4]], got[4]

    def assert_equal(self, got, fo, want, coded, what):
        """Every utterance's frames of the packed rows equal its padded rows (full rows: its fft_size / 2 + 1)."""
        c = self.c
        assert fo[0] == 0 and list(np.diff(fo)) == c.frames, what
        for u, F in enumerate(c.frames):
            a = fo[u]
            bins = DIMS if coded else c.sizes[u] // 2 + 1
            for name, g, w in zip(("time axis", "f0"), got[:2], want[:2]):
                assert np.array_equal(g[a:a + F], w[u, :F]), f"{what}: {name}, utterance {u}"
            for name, g, w in zip(("spectrogram", "aperiodicity"), got[2:], want[2:]):
                k = bins if name == "spectrogram" else (w.shape[-1] if coded else bins)
                assert np.array_equal(g[a:a + F, :k], w[u, :F, :k]), f"{what}: {name}, utterance {u}"


def check_equal(world, fs, n_samples, n_utts, method="harvest", f0_options=True, spectral_options=True):
    """Device and host, full and coded rows (nbit 0, 16 and 24 for the coded ones): bit for bit the padded chain's."""
    P = Packed(world, fs, n_samples, n_utts, method=method, f0_options=f0_options, spectral_options=spectral_options)
    for host in (False, True):
        want = P.padded(world, host=host)
        got, fo = P.packed(world, host=host)
        P.assert_equal(got, fo, want, False, f"full rows, host={host}")
        assert np.array_equal(fo, world.packed_frames(fs, P.xo, 5.0))
        for nbit in (0, 16, 24):
            want = P.padded(world, coded=True, nbit=nbit, host=host)
            got, fo = P.packed(world, coded=True, nbit=nbit, host=host)
            P.assert_equal(got, fo, want, True, f"coded rows, nbit {nbit}, host={host}")
    assert (got[1] > 0).sum() > 20


def check_edges(world, fs, n_samples):
    """Utterances of 1 and 2 samples, and shorter than one frame period, among ordinary ones; one utterance; none."""
    short = fs * 3 // 1000   # 3 ms: one frame
    lens = [n_samples, 1, short, n_samples // 2, 2, n_samples * 3 // 4]
    P = Packed(world, fs, n_samples, len(lens), lens=lens, seed=22)
    for host in (False, True):
        P.assert_equal(*P.packed(world, host=host), P.padded(world, host=host), False, f"edges, host={host}")
        P.assert_equal(*P.packed(world, coded=True, nbit=16, host=host), P.padded(world, coded=True, nbit=16, host=host),
                       True, f"edges coded, host={host}")
    one = Packed(world, fs, n_samples, 1, seed=23)
    one.assert_equal(*one.packed(world), one.padded(world), False, "one utterance")
    one.assert_equal(*one.packed(world, host=True), one.padded(world, host=True), False, "one utterance, host")
    ao = world.analysis_option(fs)
    for got in (world.analyze_packed(pc.make(world, np.zeros(1)), [0], fs, ao),
                world.analyze_host_packed(np.zeros(1), [0], fs, ao),
                world.analyze_coded_packed(pc.make(world, np.zeros(1)), 0, [0], fs, ao, DIMS),
                world.analyze_coded_host_packed(np.zeros(1), 0, [0], fs, ao, DIMS)):
        assert list(got[4]) == [0] and got[1].shape[0] == 0
    assert list(world.packed_frames(fs, [0], 5.0)) == [0]


def slice_bytes(lens, frames):
    """The padded rows of one lane slice over these utterances (packed_run's rule): offsets, samples, time axis, f0."""
    m = len(lens)
    return 16 * (m + 1) + m * (max(lens) * 8 + max(frames) * 16)


def check_long_among_short(world, fs, long_n, short_n, n_short, budget):
    """One long utterance among many short ones, with a scratch budget whose quarter cannot hold the padded rows of
    the slices cut by samples: the slices are halved, and every row is still the padded chain's."""
    from world_b200.api import World
    k = n_short // 3
    lens = [short_n] * k + [long_n] + [short_n] * (n_short - k)
    P = Packed(world, fs, long_n, len(lens), lens=lens, seed=24)
    half = len(lens) // 2
    assert slice_bytes(lens[:half], P.c.frames[:half]) > budget // 4   # the slice of the long utterance splits
    assert slice_bytes([long_n], P.c.frames[k:k + 1]) <= budget // 4
    want = P.padded(world)
    small = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    small.set_scratch_budget(budget)
    P.assert_equal(*P.packed(small), want, False, "split slices")
    P.assert_equal(*P.packed(small, host=True), P.padded(world, host=True), False, "split slices, host")


def check_slices_and_chunks(world, fs, n_samples, n_utts):
    """The rows are identical whatever the lane slices (1, 2 or 5); the host chain gives them with the smallest
    scratch budget (the stages chunk inside a slice) and chunks of three utterances."""
    from world_b200.api import World
    P = Packed(world, fs, n_samples, n_utts, seed=25)
    want = P.padded(world)
    for s in (1, 2, 5):
        with cs._Env(WB_LANE_SLICES=s):
            P.assert_equal(*P.packed(world), want, False, f"{s} lane slices")
            P.assert_equal(*P.packed(world, coded=True), P.padded(world, coded=True), True, f"{s} slices, coded")
    small = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    small.set_scratch_budget(SMALL_BUDGET)
    with cs._Env(WB_HOST_CHUNK=3, WB_HOST_SUB=2):
        P.assert_equal(*P.packed(small, host=True), want, False, "host chunks, small budget")
        P.assert_equal(*P.packed(small, coded=True, nbit=16, host=True), P.padded(world, coded=True, nbit=16), True,
                       "host chunks, coded")
    P.assert_equal(*P.packed(small), want, False, "device, small budget")


def check_bounds(world, fs, n_samples, n_utts=5, guard=3):
    """Outputs with guard frames past F and rows wider than needed, all NaN: a device call leaves the guard frames and
    the tail of each row past fft_size / 2 + 1 as they were; a host call writes F frames with zeros in that tail."""
    P = Packed(world, fs, n_samples, n_utts, seed=26)
    c = P.c
    F, W = sum(c.frames), c.width + 3
    for host in (False, True):
        mk = (lambda a: a) if host else (lambda a: pc.make(world, a))
        out = dict(time_axis=mk(np.full(F + guard, np.nan)), f0=mk(np.full(F + guard, np.nan)),
                   spectrogram=mk(np.full((F + guard, W), np.nan)), aperiodicity=mk(np.full((F + guard, W), np.nan)))
        got, fo = P.packed(world, host=host, **out)
        P.assert_equal(got, fo, P.padded(world, host=host), False, f"bounds, host={host}")
        for name, g in zip(("time axis", "f0", "spectrogram", "aperiodicity"), got):
            assert np.isnan(g[F:]).all(), f"{name} guard frames, host={host}"
        for u in range(n_utts):
            bins = c.sizes[u] // 2 + 1
            for name, g in zip(("spectrogram", "aperiodicity"), got[2:]):
                tail = g[fo[u]:fo[u + 1], bins:]
                assert (not tail.any()) if host else np.isnan(tail).all(), f"{name} tail, utterance {u}, host={host}"
        coded = dict(time_axis=mk(np.full(F + guard, np.nan)), f0=mk(np.full(F + guard, np.nan)),
                     coded_sp=mk(np.full((F + guard, DIMS), np.nan)),
                     coded_ap=mk(np.full((F + guard, world.number_of_aperiodicities(fs)), np.nan)))
        got, fo = P.packed(world, coded=True, host=host, **coded)
        for name, g in zip(("time axis", "f0", "coded sp", "coded ap"), got):
            assert np.isfinite(g[:F]).all() and np.isnan(g[F:]).all(), f"coded {name}, host={host}"


def check_vs_ref(world, ref, fs, n_samples, n_utts=4):
    """A few utterances of the packed device chain within the reference's tolerance of its own chain at their
    options (Harvest at the speaker's range, CheapTrick and D4C at its size and threshold)."""
    P = Packed(world, fs, n_samples, n_utts, seed=27)
    c = P.c
    (t, f0, sp, ap), fo = P.packed(world)
    for u in range(n_utts):
        k, fft, a, b = c.speaker[u], c.sizes[u], fo[u], fo[u + 1]
        xu = np.ascontiguousarray(c.x[u, :c.lens[u]])
        ro = ref.harvest_option()
        ro.f0_floor, ro.f0_ceil = FLOORS[k], 800.0
        tr, fr = ref.harvest(xu, fs, ro)
        co = ref.cheaptrick_option(fs)
        co.f0_floor, co.fft_size = FLOORS[k], fft
        do = ref.d4c_option()
        do.threshold = cs.THRESHOLDS[k]
        assert b - a == len(fr)
        assert np.array_equal(t[a:b], tr), f"time axis, utterance {u}"
        assert not ((f0[a:b] > 0) != (fr > 0)).any(), f"V/UV flip, utterance {u}"
        assert rel_err(f0[a:b], fr).max() <= pc.TOL, f"f0, utterance {u}"
        pc.assert_close(sp[a:b, :fft // 2 + 1], ref.cheaptrick(xu, fs, tr, fr, co), f"spectrogram utt {u}")
        pc.assert_close(ap[a:b, :fft // 2 + 1], ref.d4c(xu, fs, tr, fr, fft, do), f"aperiodicity utt {u}")


def _raises(world, fn, pattern, utt=None):
    with pytest.raises(WorldError, match=r"error 3"):
        fn()
    msg = world.lib.world_b200_last_error(world._h).decode()
    assert pattern in msg, msg
    if utt is not None:
        assert f"utterance {utt})" in msg, msg


def check_invalid(world, fs=16000):
    """Each EINVAL rule names its first bad utterance and leaves the outputs and f_offsets as they were."""
    P = Packed(world, fs, fs // 4, 4, seed=28)
    c = P.c
    data, _ = P.x_packed()
    xd = pc.make(world, data)
    F, W = sum(c.frames), c.width
    sent = [np.full(F, 7.0), np.full(F, 7.0), np.full((F, W), 7.0), np.full((F, W), 7.0)]
    dev = [pc.make(world, a) for a in sent]
    host = [a.copy() for a in sent]
    names = ("time_axis", "f0", "spectrogram", "aperiodicity")
    coded_dev = [dev[0], dev[1], pc.make(world, np.full((F, DIMS), 7.0)), pc.make(world, np.full((F, 1), 7.0))]

    def calls(xo=P.xo, kw=c.kw, ao=c.ao, dims=DIMS, dev_rows=dev, host_rows=host):
        return (lambda: world.analyze_packed(xd, xo, fs, ao, **dict(zip(names, dev_rows)), **kw),
                lambda: world.analyze_host_packed(data, xo, fs, ao, **dict(zip(names, host_rows)), **kw),
                lambda: world.analyze_coded_packed(xd, 0, xo, fs, ao, dims, time_axis=coded_dev[0], f0=coded_dev[1],
                                                   coded_sp=coded_dev[2], coded_ap=coded_dev[3], **kw))

    xo = P.xo
    bad_offsets = [(np.concatenate([[1], xo[1:]]), "x_offsets[0]", None),
                   (np.array([0, xo[1], xo[1] - 5, xo[3], xo[4]]), "x_offsets must increase", 1),
                   (np.array([0, xo[1], xo[2], xo[2], xo[4]]), "x_offsets must increase", 2),
                   (np.array([0, xo[1], xo[1] + 2 ** 31, xo[1] + 2 ** 31 + 5, xo[1] + 2 ** 31 + 9]),
                    "INT_MAX", 1)]
    for offs, pattern, u in bad_offsets:
        for fn in calls(xo=offs):
            _raises(world, fn, pattern, u)
        with pytest.raises(WorldError):
            world.packed_frames(fs, offs, 5.0)
    # NULL offsets, straight through the C ABI
    ptr = lambda a: a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data   # noqa: E731
    for name, x, rows in (("world_b200_analyze_packed", xd, dev), ("world_b200_analyze_host_packed", data, host)):
        rc = getattr(world.lib, name)(world._h, ptr(x), 4, None, fs, C.byref(c.ao), None, None, None, None,
                                      ptr(rows[0]), ptr(rows[1]), 0, ptr(rows[2]), ptr(rows[3]), None)
        assert rc == 3 and "x_offsets must be given" in world.lib.world_b200_last_error(world._h).decode()

    def with_option(name, u, field, value):
        kw = {k: list(v) for k, v in c.kw.items()}
        o = type(kw[name][u]).from_buffer_copy(kw[name][u])
        setattr(o, field, value)
        kw[name][u] = o
        return kw

    for kw, pattern, u in [(with_option("cheaptrick_options", 2, "fft_size", 1000), "power of two", 2),
                           (with_option("d4c_options", 1, "threshold", float("inf")), "threshold", 1),
                           (with_option("harvest_options", 3, "frame_period", 4.0), "frame_period", 3)]:
        for fn in calls(kw=kw):
            _raises(world, fn, pattern, u)
    # per-utterance DIO options on a Harvest chain
    dio_kw = {k: v for k, v in c.kw.items() if k != "harvest_options"}
    import dio_ranges_common as dr
    dio_kw["dio_options"] = dr.options([(40.0, 800.0, 2.0, 0.1)] * 4)
    for fn in calls(kw=dio_kw):
        _raises(world, fn, "DIO")
    # a row_stride below an utterance's fft_size / 2 + 1 names the first utterance of the largest size
    narrow_dev = [dev[0], dev[1], pc.make(world, sent[2][:, :W - 1]), pc.make(world, sent[3][:, :W - 1])]
    narrow_host = [host[0], host[1], sent[2][:, :W - 1].copy(), sent[3][:, :W - 1].copy()]
    for fn in calls(dev_rows=narrow_dev, host_rows=narrow_host)[:2]:
        _raises(world, fn, "row_stride", c.sizes.index(max(c.sizes)))
    # number_of_dimensions against every utterance's size names the first utterance at the smallest size
    _raises(world, calls(dims=min(c.sizes) // 4 + 2)[2], "number_of_dimensions", c.sizes.index(min(c.sizes)))
    world.synchronize()
    for name, want, d, h in zip(names, sent, dev, host):
        assert np.array_equal(pc.to_np(d), want) and np.array_equal(h, want), name
    for a in coded_dev[2:] + narrow_dev[2:] + narrow_host[2:]:
        assert (pc.to_np(a) == 7.0).all()
    # the context keeps working
    got, fo = P.packed(world)
    P.assert_equal(got, fo, P.padded(world), False, "after the rejections")
