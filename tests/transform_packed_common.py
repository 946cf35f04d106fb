"""Checks of the packed voice transformation (world_b200_transform_packed, world_b200_transform_host_packed and
world_b200_transform_packed_samples): utterances back to back in with n + 1 sample offsets, transformed samples back to
back out with n + 1 sample offsets.  The oracle is the padded transform (world_b200_transform_batch_spectral_options, or
world_b200_transform_batch without spectral options) on the same utterances, which transform_common.py ties to the
stepwise chain and the reference demo: every utterance's output segment must equal its padded row bit for bit.  The
same assertions run against the host emulation (CPU) and the CUDA library (-m gpu)."""
import ctypes as C
import os

import numpy as np

import packed_common as pk
import packed_synthesis_common as ps
import test_parity_common as pc
import transform_common as tc
from test_stage_paths import SMALL_BUDGET, _with_budget

EINVAL = 3
SCALES = [1.2, 0.8, 1.5, 0.9, 1.1, 0.7]
RATIOS = [1.1, 0.9, 1.0, 1.2, 0.95, 1.05]
# (nbit in, nbit out, factors): every input width, both outputs and the three factor families
COMBOS = [(0, 0, "both"), (16, 16, "f0"), (24, 0, "none"), (16, 0, "both"), (24, 16, "f0")]


def factors(n, family):
    """(f0_scale, spectral_ratio) of a factor family: "none", "f0" (f0_scale only) or "both"."""
    scale = [SCALES[u % len(SCALES)] for u in range(n)]
    ratio = [RATIOS[u % len(RATIOS)] for u in range(n)]
    return {"none": (None, None), "f0": (scale, None), "both": (scale, ratio)}[family]


def time_scales(n):
    """time_scale mixed per utterance from transform_common.TIME_SCALES."""
    return [tc.TIME_SCALES[(u + 1) % len(tc.TIME_SCALES)] for u in range(n)]


class Case:
    """A packed batch of packed_common (interleaved CheapTrick sizes and per-speaker options where spectral_options,
    per-utterance F0 ranges where f0_options), its padded rows, and one set of factors; x replaces the signals."""

    def __init__(self, world, fs, n_samples, n_utts, method="harvest", f0_options=True, spectral_options=True,
                 lens=None, seed=41, family="both", tscales=True, x=None, fft=None):
        P = pk.Packed(world, fs, n_samples, n_utts, method=method, f0_options=f0_options, seed=seed, lens=lens,
                      spectral_options=spectral_options)
        c = P.c
        if x is not None:
            c.x[:] = 0.0
            for u, m in enumerate(c.lens):
                c.x[u, :m] = x[u][:m]
        if fft is not None:
            c.ao = tc.option(world, fs, method, fft)
        self.P, self.c, self.fs, self.n = P, c, fs, n_utts
        self.xo = P.xo
        self.scale, self.ratio = factors(n_utts, family)
        self.tscales = time_scales(n_utts) if tscales else None
        self.fp = tc.frame_period(c.ao)

    def kw(self):
        return dict(f0_scale=self.scale, spectral_ratio=self.ratio, time_scale=self.tscales, **self.c.kw)

    def padded(self, world, nbit, nbit_out):
        """The padded transform's rows [n, max y_length] (host) and y_lengths."""
        _, rows = self.P.x_packed(nbit)
        X = pc.make(world, rows, rows.dtype)
        y, yl = world.transform(X, nbit, self.fs, self.c.ao, x_lengths=self.c.lens,
                                dtype="int16" if nbit_out == 16 else None, **self.kw())
        world.synchronize()
        return pc.to_np(y), yl

    def packed(self, world, nbit, nbit_out):
        """The packed device call into y with guard samples: (y [Y] host, y_offsets, guards untouched)."""
        data, _ = self.P.x_packed(nbit)
        yo = world.transform_packed_samples(self.fs, self.xo, self.fp, self.tscales)
        Y = int(yo[-1])
        fill = -12345 if nbit_out == 16 else np.nan
        yg, y = ps.guarded(world, np.zeros(Y), fill, np.int16 if nbit_out == 16 else np.float64)
        got, go = world.transform_packed(pc.make(world, data, data.dtype), nbit, self.xo, self.fs, self.c.ao,
                                         dtype="int16" if nbit_out == 16 else None, y=y, **self.kw())
        world.synchronize()
        assert got is y and np.array_equal(go, yo), "y_offsets differ from transform_packed_samples"
        return pc.to_np(y), go, ps.untouched(yg, fill)

    def host(self, world, nbit, nbit_out, pinned=False):
        """The packed host call into an out array with guard samples: (y [Y], y_offsets, guards untouched)."""
        data, _ = self.P.x_packed(nbit)
        Y = int(world.transform_packed_samples(self.fs, self.xo, self.fp, self.tscales)[-1])
        dt = np.int16 if nbit_out == 16 else np.float64
        fill = -12345 if nbit_out == 16 else 7.0
        if pinned:
            import torch
            xin = torch.from_numpy(np.ascontiguousarray(data)).pin_memory()
            buf = torch.full((Y + 2 * ps.GUARD,), fill, dtype=torch.int16 if nbit_out == 16 else torch.float64)
            buf = buf.pin_memory()
            out = buf[ps.GUARD:ps.GUARD + Y]
        else:
            xin = data
            buf = np.full(Y + 2 * ps.GUARD, fill, dtype=dt)
            out = buf[ps.GUARD:ps.GUARD + Y]
        got, go = world.transform_host_packed(xin, nbit, self.xo, self.fs, self.c.ao,
                                              dtype="int16" if nbit_out == 16 else None, out=out, **self.kw())
        b = pc.to_np(buf)
        clean = (b[:ps.GUARD] == fill).all() and (b[ps.GUARD + Y:] == fill).all()
        return pc.to_np(got), go, clean

    def assert_equal(self, got, yo, want, yl, what):
        """Every utterance's segment of the packed output equals its padded row, bit for bit."""
        assert list(np.diff(yo)) == list(yl), f"{what}: y_offsets do not follow the padded y_lengths"
        assert len(got) == yo[-1]
        for u in range(self.n):
            assert np.array_equal(got[yo[u]:yo[u + 1]], want[u, :yl[u]]), f"{what}: utterance {u} differs"
        assert np.abs(got.astype(np.float64)).max() > 0, f"{what}: silent"


def check_equal(world, fs, n_samples, n_utts, method="harvest", f0_options=True, spectral_options=True,
                combos=COMBOS):
    """The device call against the padded transform for each (nbit in, nbit out, factor family) of combos; guard
    samples on either side of y stay untouched."""
    for nbit, nbit_out, family in combos:
        K = Case(world, fs, n_samples, n_utts, method=method, f0_options=f0_options,
                 spectral_options=spectral_options, family=family)
        want, yl = K.padded(world, nbit, nbit_out)
        got, yo, clean = K.packed(world, nbit, nbit_out)
        what = f"nbit {nbit} -> {nbit_out}, factors {family}"
        assert clean, f"{what}: samples outside [0, Y) were written"
        K.assert_equal(got, yo, want, yl, what)


def check_host(world, fs=16000, n_samples=3200, n_utts=5, pinned=(False,)):
    """The host call equals the device call bit for bit, float64 and int16 out, at the default chunks, one utterance
    per chunk and two per chunk; exactly Y samples are written."""
    K = Case(world, fs, n_samples, n_utts, family="both")
    old = os.environ.get("WB_HOST_CHUNK")
    try:
        for nbit, nbit_out in ((16, 16), (0, 0)):
            os.environ.pop("WB_HOST_CHUNK", None)
            want, wo, _ = K.packed(world, nbit, nbit_out)
            for chunk in (None, "1", "2"):
                if chunk:
                    os.environ["WB_HOST_CHUNK"] = chunk
                else:
                    os.environ.pop("WB_HOST_CHUNK", None)
                for pin in pinned:
                    got, go, clean = K.host(world, nbit, nbit_out, pinned=pin)
                    what = f"nbit {nbit} -> {nbit_out}, chunk {chunk}, pinned {pin}"
                    assert clean, f"{what}: the host call wrote outside its Y samples"
                    assert np.array_equal(go, wo) and np.array_equal(got, want), f"{what}: host differs from device"
    finally:
        if old is None:
            os.environ.pop("WB_HOST_CHUNK", None)
        else:
            os.environ["WB_HOST_CHUNK"] = old


def slice_rows(world, fs, lens, fft):
    """A slice's buffer over these utterances (transform_packed_run's rule): offsets, padded samples, time axis and f0
    as long as its longest utterance, then packed f0, spectrogram and aperiodicity frames."""
    up = lambda b: (b + 255) // 256 * 256   # noqa: E731
    frames = [world.frames(fs, m, 5.0) for m in lens]
    m, row = len(lens), fft // 2 + 1
    F = sum(frames)
    return (up(16 * (m + 1)) + up(m * max(lens) * 8) + 2 * up(m * max(frames) * 8) + up(F * 8) +
            2 * up(F * row * 8))


def check_slices(world, fs, seconds, n_utts, fft, one_per_slice):
    """At the smallest budget the batch runs in more slices than by default (one utterance each where one_per_slice),
    with the same samples, equal to the padded transform."""
    n = int(seconds * fs)
    lens = [n - 997 * u for u in range(n_utts)]
    K = Case(world, fs, n, n_utts, method="dio", f0_options=False, spectral_options=False, lens=lens, fft=fft)
    lanes = 1 if world.xp == "numpy" else 2
    cap = SMALL_BUDGET // lanes // 2
    pairs = [slice_rows(world, fs, lens[u:u + 2], fft) for u in range(n_utts - 1)]
    if one_per_slice:
        assert min(pairs) > cap, "two utterances fit one slice"
    else:
        assert max(pairs) <= cap < slice_rows(world, fs, lens, fft), "the batch does not need several slices"
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs, launches = [], []
        for w in (world, small):
            before = w.launch_count()
            outs.append(K.packed(w, 16, 16))
            launches.append(w.launch_count() - before)
    finally:
        small.close()
    assert launches[1] > launches[0], f"launches: {launches[0]} by default, {launches[1]} at the small budget"
    assert outs[1][2] and np.array_equal(outs[0][0], outs[1][0]), "the sliced result differs"
    want, yl = K.padded(world, 16, 16)
    K.assert_equal(outs[1][0], outs[1][1], want, yl, "sliced")


def check_long_among_short(world, fs, long_n, short_n, n_short, fft=None):
    """One long utterance among many short ones at the smallest budget, so the slices split: equal to the padded
    transform, in more slices than by default."""
    lens = [short_n] * (n_short + 1)
    lens[n_short // 3] = long_n
    K = Case(world, fs, long_n, n_short + 1, lens=lens, seed=43, fft=fft)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        base = world.launch_count()
        got0, yo0, _ = K.packed(world, 16, 16)
        default = world.launch_count() - base
        base = small.launch_count()
        got, yo, clean = K.packed(small, 16, 16)
        sliced = small.launch_count() - base
    finally:
        small.close()
    assert clean and np.array_equal(got, got0), "the result at the smallest budget differs"
    assert sliced > default, f"launches: {default} by default, {sliced} at the smallest budget: no more slices"
    want, yl = K.padded(world, 16, 16)
    K.assert_equal(got, yo, want, yl, "long among short")


def check_relaid(world, fs=16000, n_samples=8000):
    """transform_common.high_tone scaled by 2 makes its pass be laid out again from its pulse counts: one more launch
    than at 1.0, and still the padded transform's samples."""
    tone = tc.high_tone(fs, n_samples)
    counts = []
    for s in (1.0, 2.0):
        K = Case(world, fs, n_samples, 2, f0_options=False, x=[tone, tone], tscales=False, family="none")
        K.scale = [s, 1.0]
        before = world.launch_count()
        got, yo, clean = K.packed(world, 0, 0)
        counts.append(world.launch_count() - before)
    assert counts[1] == counts[0] + 1, f"launches {counts}: the pass was not laid out again"
    want, yl = K.padded(world, 0, 0)
    assert clean
    K.assert_equal(got, yo, want, yl, "relaid pass")


def check_edges(world, fs=16000, n_samples=3200):
    """An utterance of exactly 2 frames among longer ones, one utterance alone, and none."""
    two = fs * 6 // 1000   # 6 ms: 2 frames at 5 ms
    assert world.frames(fs, two, 5.0) == 2
    lens = [n_samples, two, n_samples // 2, two]
    K = Case(world, fs, n_samples, len(lens), lens=lens, seed=44)
    want, yl = K.padded(world, 16, 0)
    got, yo, clean = K.packed(world, 16, 0)
    assert clean
    K.assert_equal(got, yo, want, yl, "2-frame utterances")
    one = Case(world, fs, n_samples, 1, seed=45)
    want, yl = one.padded(world, 0, 16)
    got, yo, clean = one.packed(world, 0, 16)
    assert clean
    one.assert_equal(got, yo, want, yl, "one utterance")
    ao = world.analysis_option(fs)
    before = world.launch_count()
    y, yo = world.transform_packed(pc.make(world, np.zeros(1)), 0, [0], fs, ao)
    yh, yoh = world.transform_host_packed(np.zeros(1), 0, [0], fs, ao)
    world.synchronize()
    assert list(yo) == [0] and list(yoh) == [0] and len(y) == 0 and len(yh) == 0
    assert world.launch_count() == before, "an empty batch queued work"
    assert list(world.transform_packed_samples(fs, [0])) == [0]


def check_samples(world, fs=22050):
    """transform_packed_samples agrees with transform_samples for each utterance, and rejects what it cannot give."""
    lens = [1, 79, 160, 22050, 12345, 3]
    xo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    for fp in (5.0, 2.5):
        for ts in (None, [0.8, 1.0, 1.25, 2.0, 0.9, 1.1]):
            yo = world.transform_packed_samples(fs, xo, fp, ts)
            want = [world.transform_samples(fs, m, fp, 1.0 if ts is None else ts[u]) for u, m in enumerate(lens)]
            assert list(np.diff(yo)) == want and yo[0] == 0, f"frame_period {fp}, time_scale {ts}"
    lib = world.lib
    good = [1.0] * len(lens)
    cases = [("x_offsets[0] = 1", [1] + list(xo[1:]), None), ("an empty utterance", [0, 5, 5, 9, 10, 11, 12], None),
             ("time_scale 0", xo, [1.0, 0.0] + good[2:]), ("time_scale NaN", xo, good[:3] + [float("nan")] + good[4:]),
             ("an output past INT_MAX", xo, good[:3] + [1e9] + good[4:])]
    for what, offs, ts in cases:
        out = (C.c_longlong * len(lens + [0]))(*([-7] * (len(lens) + 1)))
        rc = lib.world_b200_transform_packed_samples(fs, len(lens), ps.off_arg(offs), 5.0,
                                                     None if ts is None else (C.c_double * len(ts))(*ts), out)
        assert rc == EINVAL, f"{what}: returned {rc}"
        assert list(out) == [-7] * (len(lens) + 1), f"{what}: y_offsets were written"


def check_invalid(world, fs=16000):
    """Every bad argument is EINVAL before anything is queued: no launch, y (device and host) untouched, y_offsets
    untouched, last_error naming the first bad utterance k."""
    n, k = 4, 2
    K = Case(world, fs, 3200, n, seed=46)
    data, _ = K.P.x_packed(16)
    X = pc.make(world, data, data.dtype)
    xo = [int(v) for v in K.xo]
    Y = int(world.transform_packed_samples(fs, xo, 5.0)[-1])
    y = pc.make(world, np.full(Y, -7.0))
    yh = np.full(Y, -7.0)
    lib = world.lib
    c = K.c
    ct = (type(c.kw["cheaptrick_options"][0]) * n)(*c.kw["cheaptrick_options"])
    d4 = (type(c.kw["d4c_options"][0]) * n)(*c.kw["d4c_options"])
    ho = (type(c.kw["harvest_options"][0]) * n)(*c.kw["harvest_options"])
    good = [1.0] * n

    def at(v, u, val):
        out = list(v)
        out[u] = val
        return out

    def d(v):
        return None if v is None else (C.c_double * len(v))(*v)

    def call(nbit=16, offs=xo, hopt=ho, cto=ct, sc=None, ra=None, ts=None, nbit_out=0, yp="y", host=False):
        fn = lib.world_b200_transform_host_packed if host else lib.world_b200_transform_packed
        xp = data.ctypes.data if host else ps.pc_ptr(X)
        out = {"y": yh.ctypes.data if host else ps.pc_ptr(y), None: None}[yp]
        return lambda: fn(world._h, xp, nbit, n, None if offs is None else ps.off_arg(offs), fs, C.byref(c.ao), hopt,
                          None, cto, d4, d(sc), d(ra), d(ts), nbit_out, out, yo_out)

    def moved(v, u, by):   # utterance u shorter or longer by `by` samples, the others as they were
        out = list(v)
        for i in range(u + 1, len(out)):
            out[i] += by
        return out

    hbad = (type(c.kw["harvest_options"][0]) * n)(*c.kw["harvest_options"])
    hbad[k].frame_period = 2.5
    cbad = (type(c.kw["cheaptrick_options"][0]) * n)(*c.kw["cheaptrick_options"])
    cbad[k].fft_size = 8192
    one_frame = fs * 4 // 1000   # 4 ms: 1 frame
    cases = [
        ("nbit 12", call(nbit=12), "nbit"),
        ("nbit_out 8", call(nbit_out=8), "nbit_out"),
        ("y NULL", call(yp=None), "y must be given"),
        ("x_offsets NULL", call(offs=None), "x_offsets must be given"),
        ("x_offsets[0] = 1", call(offs=at(xo, 0, 1)), "x_offsets[0]"),
        ("an empty utterance", call(offs=moved(xo, k, -(xo[k + 1] - xo[k]))), f"utterance {k})"),
        ("one frame", call(offs=moved(xo, k, one_frame - (xo[k + 1] - xo[k]))), f"utterance {k})"),
        ("fft_size 8192", call(cto=cbad), f"utterance {k})"),
        ("harvest options: frame_period differs", call(hopt=hbad), f"utterance {k}"),
        ("an output past INT_MAX", call(ts=at(good, k, 1e9)), f"utterance {k}"),
        ("host: time_scale -1", call(ts=at(good, k, -1.0), host=True), f"time_scale[{k}]"),
        ("host: nbit_out 8", call(nbit_out=8, host=True), "nbit_out"),
    ]
    for what, v in (("0", 0.0), ("-1", -1.0), ("NaN", float("nan")), ("inf", float("inf"))):
        cases.append((f"time_scale {what}", call(ts=at(good, k, v)), f"time_scale[{k}]"))
        cases.append((f"f0_scale {what}", call(sc=at(good, k, v)), f"f0_scale[{k}]"))
        cases.append((f"spectral_ratio {what}", call(ra=at(good, k, v)), f"spectral_ratio[{k}]"))
    yo_out = (C.c_longlong * (n + 1))(*([-7] * (n + 1)))
    for what, fn, named in cases:
        world._use_current_stream()
        before = world.launch_count()
        rc = fn()
        world.synchronize()
        err = lib.world_b200_last_error(world._h).decode()
        assert rc == EINVAL, f"{what}: returned {rc}"
        assert world.launch_count() == before, f"{what}: kernels were launched"
        assert named in err, f"{what}: last_error {err!r} does not name {named!r}"
        assert (pc.to_np(y) == -7.0).all() and (yh == -7.0).all(), f"{what}: y was written"
        assert list(yo_out) == [-7] * (n + 1), f"{what}: y_offsets were written"
    rc = call()()
    world.synchronize()
    assert rc == 0 and not (pc.to_np(y) == -7.0).all(), "the context does not work after the errors"
    assert list(yo_out) == [int(v) for v in world.transform_packed_samples(fs, xo, 5.0)]
