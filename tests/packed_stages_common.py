"""Checks of the packed stage calls (world_b200_stonemask_packed, *_cheaptrick_*packed, *_d4c_*packed and the packed
codec): utterances back to back with n + 1 sample offsets, frames back to back with the caller's n + 1 frame offsets.
Each utterance's output is compared bit for bit with the padded _options call (or the padded *_batch codec call at its
size) on the same utterance; the same assertions run against the host emulation (CPU) and the CUDA library (-m gpu)."""
import ctypes as C

import numpy as np
import pytest

import packed_common as pk
import test_parity_common as pc
from refworld import rel_err
from world_b200.api import WorldError

DIMS = pk.DIMS


def padded(a, fo, width=None):
    """Packed frames [F(, W)] -> padded rows [n, L(, W)] (zeros past each utterance's frames)."""
    a = pc.to_np(a)
    F = np.diff(fo)
    L = max(1, int(F.max()) if len(F) else 1)
    out = np.zeros((len(F), L) + a.shape[1:])
    for u, n in enumerate(F):
        out[u, :n] = a[fo[u]:fo[u] + n]
    return out


class Stages:
    """A packed case of packed_common (two CheapTrick sizes, per-speaker D4C thresholds) with its chain's F0, or an
    external F0 at another hop (ext_hop ms): unvoiced stretches and frames below CheapTrick's floor included."""

    def __init__(self, world, fs, n_samples, n_utts, method="harvest", lens=None, seed=31, ext_hop=None):
        self.P = P = pk.Packed(world, fs, n_samples, n_utts, method=method, lens=lens, seed=seed)
        self.world, self.fs, self.c = world, fs, P.c
        self.xo = P.xo
        data, _ = P.x_packed()
        self.x = pc.make(world, data)
        self.chain, self.fo = P.packed(world)            # analyze_packed's rows: the composition's yardstick
        t, f0 = self.chain[0], self.chain[1]
        if ext_hop is not None:
            rng = np.random.default_rng(seed)
            counts = [int(1000.0 * n / fs / ext_hop) + 1 for n in self.c.lens]
            fo = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
            t = np.concatenate([np.arange(k) * ext_hop / 1000.0 for k in counts])
            f0 = np.concatenate([np.interp(np.arange(k) * ext_hop / 1000.0,
                                           self.chain[0][self.fo[u]:self.fo[u + 1]],
                                           self.chain[1][self.fo[u]:self.fo[u + 1]]) for u, k in enumerate(counts)])
            f0[rng.random(f0.shape[0]) < 0.15] = 0.0      # unvoiced frames
            f0[rng.random(f0.shape[0]) < 0.1] = 30.0      # below every floor: CheapTrick's 500 Hz stand-in
            self.fo = fo
        self.t_np, self.f0_np = np.asarray(t, dtype=np.float64), np.asarray(f0, dtype=np.float64)
        self.t, self.f0 = pc.make(world, self.t_np), pc.make(world, self.f0_np)
        self.frames = list(np.diff(self.fo))
        self.ct = self.c.kw["cheaptrick_options"]
        self.d4 = self.c.kw["d4c_options"]
        self.sizes = self.c.sizes
        # the padded counterparts' inputs
        self.x_rows = pc.make(world, self.c.x)
        self.t_rows = pc.make(world, padded(self.t_np, self.fo))
        self.f0_rows = pc.make(world, padded(self.f0_np, self.fo))

    def pad_kw(self):
        return dict(x_lengths=self.c.lens, f0_lengths=self.frames)

    def assert_rows(self, got, want, widths, what):
        """Utterance u's packed rows equal its padded rows, its first widths[u] values."""
        got, want = pc.to_np(got), pc.to_np(want)
        for u, F in enumerate(self.frames):
            a, k = self.fo[u], widths[u] if widths else None
            g = got[a:a + F] if got.ndim == 1 else got[a:a + F, :k]
            w = want[u, :F] if want.ndim == 2 else want[u, :F, :k]
            assert np.array_equal(g, w), f"{what}: utterance {u}"

    def bins(self):
        return [s // 2 + 1 for s in self.sizes]

    # the calls
    def stonemask(self, world=None, f0=None):
        w = world or self.world
        return w.stonemask_packed(self.x, self.xo, self.fs, self.t, self.f0 if f0 is None else f0, self.fo)

    def cheaptrick(self, world=None, coded=False, **kw):
        w = world or self.world
        if coded:
            return w.cheaptrick_coded_packed(self.x, self.xo, self.fs, self.t, self.f0, self.fo, DIMS, self.ct, **kw)
        return w.cheaptrick_packed(self.x, self.xo, self.fs, self.t, self.f0, self.fo, self.ct, **kw)

    def d4c(self, world=None, coded=False, **kw):
        w = world or self.world
        if coded:
            return w.d4c_coded_packed(self.x, self.xo, self.fs, self.t, self.f0, self.fo, self.sizes, self.d4, **kw)
        return w.d4c_packed(self.x, self.xo, self.fs, self.t, self.f0, self.fo, self.sizes, self.d4, **kw)

    def check_stages(self, what, stonemask=True):
        """Every packed stage call equals the padded _options call of its family, utterance by utterance (StoneMask
        only up to 48 kHz, its limit)."""
        w, kw = self.world, self.pad_kw()
        n_ap = w.number_of_aperiodicities(self.fs)
        got = self.cheaptrick()
        want = w.cheaptrick(self.x_rows, self.fs, self.t_rows, self.f0_rows, self.ct, **kw)
        self.assert_rows(got, want, self.bins(), f"{what}: cheaptrick")
        got = self.cheaptrick(coded=True)
        want = w.cheaptrick_coded(self.x_rows, self.fs, self.t_rows, self.f0_rows, DIMS, self.ct, **kw)
        self.assert_rows(got, want, [DIMS] * len(self.sizes), f"{what}: cheaptrick coded")
        got = self.d4c()
        want = w.d4c(self.x_rows, self.fs, self.t_rows, self.f0_rows, self.sizes, self.d4, **kw)
        self.assert_rows(got, want, self.bins(), f"{what}: d4c")
        if n_ap > 0:
            got = self.d4c(coded=True)
            want = w.d4c_coded(self.x_rows, self.fs, self.t_rows, self.f0_rows, self.sizes, self.d4, **kw)
            self.assert_rows(got, want, [n_ap] * len(self.sizes), f"{what}: d4c coded")
        if stonemask:
            got = self.stonemask()
            want = w.stonemask(self.x_rows, self.fs, self.t_rows, self.f0_rows, **kw)
            self.assert_rows(got, want, None, f"{what}: stonemask")
        w.synchronize()


def check_equal(world, fs, n_samples, n_utts, method="harvest", ext_hop=None):
    """Bit for bit the padded _options calls: on the chain's F0 (DIO or Harvest), or on an external F0 at another hop.
    Above 48.1 kHz D4C's transform outgrows its fast body kernel and every selected frame takes the frame list."""
    S = Stages(world, fs, n_samples, n_utts, method=method, ext_hop=ext_hop)
    S.check_stages(f"{method}, fs {fs}, hop {ext_hop}", stonemask=fs <= 48000)
    assert (S.f0_np > 0).sum() > 10


def check_composition(world, fs, n_samples, n_utts, method="harvest"):
    """analyze_packed's F0, then the packed stage calls: analyze_packed's own rows (and analyze_coded_packed's); for DIO
    the raw DIO F0 through stonemask_packed is the chain's F0."""
    S = Stages(world, fs, n_samples, n_utts, method=method)
    bins = S.bins()
    S.assert_rows(S.cheaptrick(), padded(S.chain[2], S.fo), bins, "composition: spectrogram")
    S.assert_rows(S.d4c(), padded(S.chain[3], S.fo), bins, "composition: aperiodicity")
    coded, fo = S.P.packed(world, coded=True)
    assert np.array_equal(fo, S.fo)
    S.assert_rows(S.cheaptrick(coded=True), padded(coded[2], fo), [DIMS] * n_utts, "composition: coded envelope")
    n_ap = world.number_of_aperiodicities(fs)
    if n_ap > 0:
        S.assert_rows(S.d4c(coded=True), padded(coded[3], fo), [n_ap] * n_utts, "composition: coded aperiodicity")
    if method == "dio":
        opts = S.c.kw.get("dio_options")
        t, f0, _ = world.dio(S.x_rows, fs, opts, x_lengths=S.c.lens)
        raw = np.concatenate([pc.to_np(f0)[u, :F] for u, F in enumerate(S.frames)])
        got = S.stonemask(f0=pc.make(world, raw))
        assert np.array_equal(pc.to_np(got), S.f0_np), "composition: DIO + stonemask_packed"
        raw_dev = pc.make(world, raw)
        world.stonemask_packed(S.x, S.xo, fs, S.t, raw_dev, S.fo, out=raw_dev)
        assert np.array_equal(pc.to_np(raw_dev), S.f0_np), "stonemask_packed in place"
    world.synchronize()


def check_codec(world, fs, n_samples, n_utts):
    """Each packed codec call equals the padded *_batch codec call at each utterance's size, and the packed round trip
    equals the padded one."""
    S = Stages(world, fs, n_samples, n_utts)
    sp, ap = S.cheaptrick(), S.d4c()
    n_ap = world.number_of_aperiodicities(fs)
    csp = world.code_spectral_envelope_packed(sp, S.fo, fs, S.sizes, DIMS)
    cap = world.code_aperiodicity_packed(ap, S.fo, fs, S.sizes)
    W = int(sp.shape[-1])
    dsp = world.decode_spectral_envelope_packed(csp, S.fo, fs, S.sizes, DIMS, row_stride=W)
    dap = world.decode_aperiodicity_packed(cap, S.fo, fs, S.sizes, row_stride=W)
    world.synchronize()
    sp_np, ap_np = pc.to_np(sp), pc.to_np(ap)
    for u, (F, fft) in enumerate(zip(S.frames, S.sizes)):
        if F == 0:
            continue
        a, b = S.fo[u], fft // 2 + 1
        row_sp = pc.make(world, sp_np[a:a + F, :b][None])
        row_ap = pc.make(world, ap_np[a:a + F, :b][None])
        want = pc.to_np(world.code_spectral_envelope(row_sp, fs, fft, DIMS))[0]
        assert np.array_equal(pc.to_np(csp)[a:a + F], want), f"code envelope, utterance {u}"
        want_d = pc.to_np(world.decode_spectral_envelope(pc.make(world, want[None]), fs, fft, DIMS))[0]
        assert np.array_equal(pc.to_np(dsp)[a:a + F, :b], want_d), f"decode envelope, utterance {u}"
        want = pc.to_np(world.code_aperiodicity(row_ap, fs, fft))[0]
        if n_ap > 0:
            assert np.array_equal(pc.to_np(cap)[a:a + F, :n_ap], want[:, :n_ap]), f"code aperiodicity, utterance {u}"
        want_d = pc.to_np(world.decode_aperiodicity(pc.make(world, want[None]), fs, fft))[0]
        assert np.array_equal(pc.to_np(dap)[a:a + F, :b], want_d), f"decode aperiodicity, utterance {u}"


def check_edges(world, fs, n_samples):
    """Utterances of 1 and 2 samples, utterances with 0 frames, one utterance, and none."""
    lens = [n_samples, 1, n_samples // 2, 2, n_samples * 3 // 4]
    S = Stages(world, fs, n_samples, len(lens), lens=lens, seed=32)
    S.check_stages("1 and 2 samples")
    # frames of the caller's own: utterances 1 and 3 get none
    keep = [F if u not in (1, 3) else 0 for u, F in enumerate(S.frames)]
    t = np.concatenate([S.t_np[S.fo[u]:S.fo[u] + k] for u, k in enumerate(keep)])
    f0 = np.concatenate([S.f0_np[S.fo[u]:S.fo[u] + k] for u, k in enumerate(keep)])
    S.fo = np.concatenate([[0], np.cumsum(keep)]).astype(np.int64)
    S.frames, S.t_np, S.f0_np = keep, t, f0
    S.t, S.f0 = pc.make(world, t), pc.make(world, f0)
    S.t_rows, S.f0_rows = pc.make(world, padded(t, S.fo)), pc.make(world, padded(f0, S.fo))
    S.check_stages("0 frames")
    one = Stages(world, fs, n_samples, 1, seed=33)
    one.check_stages("one utterance")
    # n_utts == 0
    x0, z = pc.make(world, np.zeros(1)), pc.make(world, np.zeros((0,)))
    assert world.stonemask_packed(x0, [0], fs, z, z, [0]).shape[0] == 0
    assert world.cheaptrick_packed(x0, [0], fs, z, z, [0], [], row_stride=3).shape[0] == 0
    assert world.cheaptrick_coded_packed(x0, [0], fs, z, z, [0], DIMS, []).shape[0] == 0
    assert world.d4c_packed(x0, [0], fs, z, z, [0], [], row_stride=3).shape[0] == 0
    assert world.d4c_coded_packed(x0, [0], fs, z, z, [0], []).shape[0] == 0
    e = pc.make(world, np.zeros((0, DIMS)))
    assert world.code_spectral_envelope_packed(pc.make(world, np.zeros((0, 3))), [0], fs, [], DIMS).shape[0] == 0
    assert world.decode_spectral_envelope_packed(e, [0], fs, [], DIMS, row_stride=3).shape[0] == 0
    world.synchronize()


def check_long_among_short(world, fs, long_n, short_n, n_short, budget):
    """One long utterance among many short ones at the smallest scratch budget: every row is the padded call's."""
    from world_b200.api import World
    k = n_short // 3
    lens = [short_n] * k + [long_n] + [short_n] * (n_short - k)
    S = Stages(world, fs, long_n, len(lens), lens=lens, seed=34)
    small = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    small.set_scratch_budget(budget)
    kw = S.pad_kw()
    S.assert_rows(S.cheaptrick(small), world.cheaptrick(S.x_rows, fs, S.t_rows, S.f0_rows, S.ct, **kw), S.bins(),
                  "long among short: cheaptrick")
    S.assert_rows(S.d4c(small), world.d4c(S.x_rows, fs, S.t_rows, S.f0_rows, S.sizes, S.d4, **kw), S.bins(),
                  "long among short: d4c")
    S.assert_rows(S.stonemask(small), world.stonemask(S.x_rows, fs, S.t_rows, S.f0_rows, **kw), None,
                  "long among short: stonemask")
    small.synchronize()


def check_bounds(world, fs, n_samples, n_utts=4, guard=3):
    """NaN guard frames past F and NaN rows wider than fft_size / 2 + 1 are left as they were by every call."""
    S = Stages(world, fs, n_samples, n_utts, seed=35)
    F, W = sum(S.frames), max(S.bins()) + 3
    n_ap = world.number_of_aperiodicities(fs)

    def nan(*shape):
        return pc.make(world, np.full(shape, np.nan))

    def check(got, width, what, full):
        g = pc.to_np(got)
        assert np.isnan(g[F:]).all(), f"{what}: guard frames"
        if full:
            for u, b in enumerate(S.bins()):
                assert np.isnan(g[S.fo[u]:S.fo[u + 1], b:]).all(), f"{what}: row tail, utterance {u}"
        assert not np.isnan(g[:F, :width] if g.ndim == 2 and not full else g[:F]).all(), what

    sp = S.cheaptrick(out=nan(F + guard, W))
    check(sp, None, "cheaptrick", True)
    ap = S.d4c(out=nan(F + guard, W))
    check(ap, None, "d4c", True)
    check(S.cheaptrick(coded=True, out=nan(F + guard, DIMS)), DIMS, "cheaptrick coded", False)
    if n_ap > 0:
        check(S.d4c(coded=True, out=nan(F + guard, n_ap)), n_ap, "d4c coded", False)
    out = nan(F + guard)
    world.stonemask_packed(S.x, S.xo, fs, S.t, S.f0, S.fo, out=out)
    assert np.isnan(pc.to_np(out)[F:]).all(), "stonemask: guard frames"
    csp = world.code_spectral_envelope_packed(sp, S.fo, fs, S.sizes, DIMS, out=nan(F + guard, DIMS))
    check(csp, DIMS, "code envelope", False)
    check(world.decode_spectral_envelope_packed(csp, S.fo, fs, S.sizes, DIMS, out=nan(F + guard, W)), None,
          "decode envelope", True)
    if n_ap > 0:
        cap = world.code_aperiodicity_packed(ap, S.fo, fs, S.sizes, out=nan(F + guard, n_ap))
        check(cap, n_ap, "code aperiodicity", False)
        check(world.decode_aperiodicity_packed(cap, S.fo, fs, S.sizes, out=nan(F + guard, W)), None,
              "decode aperiodicity", True)
    world.synchronize()


def check_vs_ref(world, ref, fs, n_samples, n_utts=3):
    """A few utterances against the reference's CheapTrick, D4C and StoneMask on the same F0."""
    S = Stages(world, fs, n_samples, n_utts, seed=36)
    sp, ap, sm = pc.to_np(S.cheaptrick()), pc.to_np(S.d4c()), pc.to_np(S.stonemask())
    world.synchronize()
    for u in range(n_utts):
        a, b = S.fo[u], S.fo[u + 1]
        x = S.c.x[u, :S.c.lens[u]]
        t, f0 = S.t_np[a:b], S.f0_np[a:b]
        o = ref.cheaptrick_option(fs)
        o.fft_size, o.q1 = S.ct[u].fft_size, S.ct[u].q1
        want = ref.cheaptrick(x, fs, t, f0, o)
        bins = S.sizes[u] // 2 + 1
        assert rel_err(sp[a:b, :bins], want).max() < 1e-6, f"cheaptrick vs reference, utterance {u}"
        d = ref.d4c_option()
        d.threshold = S.d4[u].threshold
        want = ref.d4c(x, fs, t, f0, S.sizes[u], d)
        assert rel_err(ap[a:b, :bins], want).max() < 1e-6, f"d4c vs reference, utterance {u}"
        want = ref.stonemask(x, fs, t, f0)
        assert rel_err(sm[a:b], want).max() < 1e-6, f"stonemask vs reference, utterance {u}"


def _raises(world, fn, pattern, utt, outs=()):
    """fn fails with EINVAL naming `pattern` (and utterance utt), before anything is queued: outs keep their NaN."""
    with pytest.raises(WorldError, match=pattern) as e:
        fn()
    if utt is not None:
        assert f"(utterance {utt})" in str(e.value), str(e.value)
    for o in outs:
        assert np.isnan(pc.to_np(o)).all(), f"output written before the check: {pattern}"


def check_invalid(world, fs=16000):
    """Every rule fails before anything is queued and names the first bad utterance; the context works afterwards."""
    S = Stages(world, fs, 3200, 4, seed=37)
    F, W = sum(S.frames), max(S.bins())
    sp = pc.make(world, np.full((F, W), np.nan))
    cs = pc.make(world, np.full((F, DIMS), np.nan))
    sm = pc.make(world, np.full((F,), np.nan))
    xo, fo = list(S.xo), list(S.fo)
    bad_x = list(xo); bad_x[2] = bad_x[1]                      # utterance 1 of 0 samples
    bad_f = list(fo); bad_f[3] = bad_f[2] - 1                  # utterance 2 of -1 frames
    shifted = [v + 1 for v in xo]                              # x_offsets[0] != 0
    ct = list(S.ct)
    bad = type(ct[0])(); C.memmove(C.byref(bad), C.byref(ct[2]), C.sizeof(bad)); bad.fft_size = 1000
    bad_ct = ct[:2] + [bad] + ct[3:]
    calls = [
        (lambda: world.cheaptrick_packed(S.x, bad_x, fs, S.t, S.f0, fo, ct, out=sp), "x_offsets", 1, [sp]),
        (lambda: world.cheaptrick_packed(S.x, shifted, fs, S.t, S.f0, fo, ct, out=sp), r"x_offsets\[0\]", None, [sp]),
        (lambda: world.d4c_packed(S.x, xo, fs, S.t, S.f0, bad_f, S.sizes, S.d4, out=sp), "f_offsets", 2, [sp]),
        (lambda: world.stonemask_packed(S.x, xo, fs, S.t, S.f0, bad_f, out=sm), "f_offsets", 2, [sm]),
        (lambda: world.cheaptrick_packed(S.x, xo, fs, S.t, S.f0, fo, bad_ct, out=sp), "power of two", 2, [sp]),
        (lambda: world.cheaptrick_packed(S.x, xo, fs, S.t, S.f0, fo, ct, row_stride=W - 1,
                                         out=pc.make(world, np.full((F, W - 1), np.nan))), "row_stride", None, []),
        (lambda: world.cheaptrick_coded_packed(S.x, xo, fs, S.t, S.f0, fo, 10000, ct, out=cs), "number_of_dimensions",
         0, [cs]),
        (lambda: world.d4c_packed(S.x, xo, fs, S.t, S.f0, fo, [S.sizes[0], 2] + S.sizes[2:], S.d4, out=sp),
         "fft_size", 1, [sp]),
        (lambda: world.code_spectral_envelope_packed(sp, bad_f, fs, S.sizes, DIMS, out=cs), "f_offsets", 2, [cs]),
        (lambda: world.code_spectral_envelope_packed(sp, fo, fs, [S.sizes[0], 100] + S.sizes[2:], DIMS, out=cs),
         "fft_size", 1, [cs]),
        (lambda: world.decode_spectral_envelope_packed(cs, fo, fs, S.sizes, DIMS, row_stride=W - 1,
                                                       out=pc.make(world, np.full((F, W - 1), np.nan))),
         "row_stride", None, []),
    ]
    for fn, pattern, utt, outs in calls:
        _raises(world, fn, pattern, utt, outs)
    # the row_stride messages name the first utterance too narrow
    with pytest.raises(WorldError, match=r"row_stride.*\(utterance \d+\)"):
        world.cheaptrick_packed(S.x, xo, fs, S.t, S.f0, fo, ct, row_stride=W - 1)
    world.synchronize()
    S.check_stages("after the errors")


def check_many_utterances(world, fs=16000, n_utts=70000, seed=38):
    """More utterances than one chunk holds (65535): one- to three-sample utterances with 0 or 1 frames, each equal to
    the padded call's, so that the chunk-relative offsets and options of every chunk are used."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 4, n_utts)
    frames = rng.integers(0, 2, n_utts)
    xo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fo = np.concatenate([[0], np.cumsum(frames)]).astype(np.int64)
    x = rng.standard_normal(int(xo[-1])) * 0.1
    F = int(fo[-1])
    t = rng.uniform(0.0, 0.0002, F)
    f0 = np.where(rng.random(F) < 0.7, rng.uniform(120.0, 400.0, F), 0.0)
    sizes = [1024 if u % 3 else 2048 for u in range(n_utts)]
    cts = []
    for k in sizes:
        o = world.cheaptrick_option(fs)
        o.fft_size = k
        cts.append(o)
    X, T, F0 = pc.make(world, x), pc.make(world, t), pc.make(world, f0)
    sp = pc.to_np(world.cheaptrick_packed(X, xo, fs, T, F0, fo, cts))
    ap = pc.to_np(world.d4c_packed(X, xo, fs, T, F0, fo, sizes))
    x_rows = np.zeros((n_utts, 3))
    t_rows, f0_rows = np.zeros((n_utts, 1)), np.zeros((n_utts, 1))
    for u in range(n_utts):
        x_rows[u, :lens[u]] = x[xo[u]:xo[u + 1]]
        t_rows[u, :frames[u]] = t[fo[u]:fo[u + 1]]
        f0_rows[u, :frames[u]] = f0[fo[u]:fo[u + 1]]
    kw = dict(x_lengths=[int(v) for v in lens], f0_lengths=[int(v) for v in frames])
    args = (pc.make(world, x_rows), fs, pc.make(world, t_rows), pc.make(world, f0_rows))
    want_sp = pc.to_np(world.cheaptrick(*args, cts, **kw))
    want_ap = pc.to_np(world.d4c(*args, sizes, **kw))
    world.synchronize()
    for u in np.flatnonzero(frames):
        b = sizes[u] // 2 + 1
        assert np.array_equal(sp[fo[u], :b], want_sp[u, 0, :b]), f"many utterances: cheaptrick, utterance {u}"
        assert np.array_equal(ap[fo[u], :b], want_ap[u, 0, :b]), f"many utterances: d4c, utterance {u}"
