"""Checks of the way back on packed rows (world_b200_synthesis_packed, world_b200_synthesis_coded_packed,
world_b200_synthesis_coded_host_packed and world_b200_modify_packed): f0 and rows as [F] frames back to back with n + 1
frame offsets, y as [Y] samples back to back with n + 1 sample offsets.  Each utterance is compared bit for bit with the
padded *_options call of the same family on the same batch; the same assertions run against the host emulation (CPU)
and the CUDA library (-m gpu)."""
import ctypes as C
import os

import numpy as np
import pytest

import synthesis_options_common as so
import test_parity_common as pc
from test_stage_paths import SMALL_BUDGET, _with_budget

FP = so.FP
GUARD = 5   # NaN (int16: a sentinel) samples and frames on either side of a packed array


def sizes_at(world, fs, n):
    """n interleaved sizes: the per-speaker CheapTrick sizes of synthesis_options_common where it has floors for fs,
    else 1024 and 2048."""
    if fs in so.FLOORS:
        return so.sizes_of(world, fs, n)
    return [(1024, 2048)[u % 2] for u in range(n)]


def offsets(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


class Packed:
    """A ragged batch of synthesis_options_common (two or three fft sizes interleaved, padding values in the rows) and
    the same utterances packed: f0 [F], full rows [F, width], coded rows [F, dims] / [F, n_ap]."""

    def __init__(self, world, fs, sizes, seconds, dims=24, seed=3, high=None, width=None, lens=None):
        b = so.Batch(world, fs, sizes, seconds, dims, seed=seed, high=high)
        if lens is not None:   # (f_len, y_len) per utterance, shorter than the batch's rows
            b.f_len, b.y_len = [v[0] for v in lens], [v[1] for v in lens]
            b.Y = max(b.y_len)
        self.b, self.n, self.fs = b, b.n, fs
        self.width = width or b.row
        self.fo, self.yo = offsets(b.f_len), offsets(b.y_len)
        self.F, self.Y = int(self.fo[-1]), int(self.yo[-1])
        cat = lambda a: np.ascontiguousarray(np.concatenate([a[u, :m] for u, m in enumerate(b.f_len)]))
        self.f0, self.csp, self.cap = cat(b.f0), cat(b.csp), cat(b.cap)
        self.sp, self.ap = cat(b.sp)[:, :self.width], cat(b.ap)[:, :self.width]
        self.sp, self.ap = np.ascontiguousarray(self.sp), np.ascontiguousarray(self.ap)

    def seg(self, y, u):
        return y[self.yo[u]:self.yo[u + 1]]


def guarded(world, a, fill=np.nan, dtype=np.float64):
    """A device (or emulation) array of a with GUARD entries of fill on either side along the first axis, and the view
    of a inside it."""
    shape = (a.shape[0] + 2 * GUARD,) + a.shape[1:]
    g = np.full(shape, fill, dtype=dtype)
    g[GUARD:GUARD + a.shape[0]] = a
    d = pc.make(world, g, dtype)
    return d, d[GUARD:GUARD + a.shape[0]]


def untouched(a, fill):
    a = pc.to_np(a)
    head, tail = a[:GUARD], a[a.shape[0] - GUARD:]
    if isinstance(fill, float) and np.isnan(fill):
        return np.isnan(head).all() and np.isnan(tail).all()
    return (head == fill).all() and (tail == fill).all()


def run_packed(world, P, family, row_stride=None):
    """The packed call of one family on P: (y as a host array, whether the guard samples stayed untouched)."""
    b, fs = P.b, P.fs
    scale, ratio = so.factors(P.n)
    if family == "host":
        fill = -12345
        y = np.full(P.Y + 2 * GUARD, fill, dtype=np.int16)
        world.synthesis_coded_host_packed(P.f0, P.csp, P.cap, P.fo, b.sizes, FP, fs, P.yo, nbit=16,
                                          out=y[GUARD:GUARD + P.Y], f0_scale=scale, spectral_ratio=ratio)
        return y[GUARD:GUARD + P.Y], (y[:GUARD] == fill).all() and (y[GUARD + P.Y:] == fill).all()
    pcm16 = family == "pcm16"
    fill = -12345 if pcm16 else np.nan
    yg, y = guarded(world, np.zeros(P.Y), fill, np.int16 if pcm16 else np.float64)
    F = pc.make(world, P.f0)
    if family == "full":
        SP, AP = pc.make(world, P.sp), pc.make(world, P.ap)
        if row_stride is None:
            world.synthesis_packed(F, SP, AP, P.fo, b.sizes, FP, fs, P.yo, y=y)
        else:   # the C call, to pass row_stride 0
            sizes = (C.c_int * P.n)(*b.sizes)
            rc = world.lib.world_b200_synthesis_packed(world._h, pc_ptr(F), P.n, off_arg(P.fo), pc_ptr(SP),
                                                       pc_ptr(AP), row_stride, sizes, FP, fs, off_arg(P.yo), pc_ptr(y))
            world._check(rc)
    else:
        kw = dict(dtype="int16") if pcm16 else {}
        if family in ("modified", "scaled"):
            kw.update(f0_scale=scale, spectral_ratio=ratio if family == "modified" else None)
        world.synthesis_coded_packed(F, pc.make(world, P.csp), pc.make(world, P.cap), P.fo, b.sizes, FP, fs, P.yo,
                                     y=y, **kw)
    world.synchronize()
    return pc.to_np(y), untouched(yg, fill)


def run_padded(world, P, family, budget_world=None):
    """The padded *_options call of the family on the same utterances, [n, Y] host rows."""
    if family == "scaled":
        w = budget_world or world
        b = P.b
        scale, _ = so.factors(P.n)
        y = w.synthesis_coded(pc.make(w, b.f0), pc.make(w, b.csp), pc.make(w, b.cap), b.sizes, FP, P.fs, b.Y,
                              f0_lengths=b.f_len, y_lengths=b.y_len, f0_scale=scale)
        w.synchronize()
        return pc.to_np(y)
    return so.run_family(world, P.b, family, budget_world=budget_world)


def assert_equal(P, got, want, what):
    for u in range(P.n):
        assert np.array_equal(P.seg(got, u), want[u, :P.b.y_len[u]]), f"{what}: utterance {u} differs"
    assert np.abs(got.astype(np.float64)).max() > 0, f"{what}: silent"


def check_full(world, fs, n=5, seconds=0.3):
    """Full rows, sizes interleaved, rows wider than every size and rows of row_stride 0 (the largest size's bins)."""
    sizes = sizes_at(world, fs, n)
    want = None
    for width in (None, max(sizes) // 2 + 1):
        P = Packed(world, fs, sizes, seconds, width=width)
        want = run_padded(world, P, "full") if want is None else want
        got, clean = run_packed(world, P, "full", row_stride=None if width is None else 0)
        assert clean, "samples outside [0, Y) were written"
        assert_equal(P, got, want, f"full rows of width {P.width}")


def check_coded(world, fs, families=("coded", "pcm16", "scaled", "modified"), n=5, seconds=0.3):
    """Coded rows, nbit 0 and 16, without factors, with f0_scale only and with both."""
    P = Packed(world, fs, sizes_at(world, fs, n), seconds)
    for family in families:
        got, clean = run_packed(world, P, family)
        assert clean, f"{family}: samples outside [0, Y) were written"
        assert_equal(P, got, run_padded(world, P, family), family)


def check_host(world, fs=16000, n=5, seconds=0.3):
    """The host packed call equals the device packed call (nbit 16, both factors): chunks of the default, of one
    utterance (WB_HOST_CHUNK=1), and at the smallest budget."""
    P = Packed(world, fs, sizes_at(world, fs, n), seconds)
    scale, ratio = so.factors(P.n)
    y = world.synthesis_coded_packed(pc.make(world, P.f0), pc.make(world, P.csp), pc.make(world, P.cap), P.fo,
                                     P.b.sizes, FP, fs, P.yo, dtype="int16", f0_scale=scale, spectral_ratio=ratio)
    world.synchronize()
    want = pc.to_np(y)
    got, clean = run_packed(world, P, "host")
    assert clean and np.array_equal(got, want), "host packed call, default chunks"
    old = os.environ.get("WB_HOST_CHUNK")
    os.environ["WB_HOST_CHUNK"] = "1"
    try:
        got, clean = run_packed(world, P, "host")
    finally:
        if old is None:
            del os.environ["WB_HOST_CHUNK"]
        else:
            os.environ["WB_HOST_CHUNK"] = old
    assert clean and np.array_equal(got, want), "host packed call, one utterance per chunk"
    small = _with_budget(world, SMALL_BUDGET)
    try:
        got, clean = run_packed(small, P, "host")
    finally:
        small.close()
    assert clean and np.array_equal(got, want), "host packed call, smallest budget"
    # the padded host call gives the same samples
    assert_equal(P, got, run_padded(world, P, "host"), "host packed call against the padded host call")


def check_modify(world, fs=16000, n=5, seconds=0.3):
    """modify_packed equals modify_batch_options per utterance; guard frames and bins past each size stay untouched."""
    P = Packed(world, fs, sizes_at(world, fs, n), seconds)
    scale, ratio = so.factors(P.n)
    want_f0, want_sp = run_padded(world, P, "modify")
    Fg, F = guarded(world, P.f0)
    Sg, S = guarded(world, P.sp)
    world.modify_packed(F, S, P.fo, fs, P.b.sizes, f0_scale=scale, spectral_ratio=ratio)
    world.synchronize()
    assert untouched(Fg, np.nan) and untouched(Sg, np.nan), "frames outside [0, F) were written"
    f0, sp = pc.to_np(F), pc.to_np(S)
    for u in range(P.n):
        a, z, bins = P.fo[u], P.fo[u + 1], P.b.sizes[u] // 2 + 1
        assert np.array_equal(f0[a:z], want_f0[u, :z - a]), f"modify_packed: f0 of utterance {u}"
        assert np.array_equal(sp[a:z, :bins], want_sp[u, :z - a, :bins]), f"modify_packed: envelope of utterance {u}"
        assert (sp[a:z, bins:] == 7.0).all(), f"modify_packed: bins past utterance {u}'s size were written"
    # row_stride 0: rows of the largest size's bins
    P0 = Packed(world, fs, P.b.sizes, seconds, width=max(P.b.sizes) // 2 + 1)
    S0 = pc.make(world, P0.sp)
    F0 = pc.make(world, P0.f0)
    sizes = (C.c_int * P.n)(*P.b.sizes)
    world._check(world.lib.world_b200_modify_packed(world._h, pc_ptr(F0), P.n, off_arg(P.fo), pc_ptr(S0), 0, sizes,
                                                    fs, (C.c_double * P.n)(*scale), (C.c_double * P.n)(*ratio)))
    world.synchronize()
    assert np.array_equal(pc.to_np(S0), sp[:, :P0.width]), "modify_packed with row_stride 0"


def check_round_trip(world, fs=16000, n=4, n_samples=4000):
    """analyze_packed -> modify_packed -> synthesis_packed equals analyze_batch (spectral options) -> modify (options)
    -> synthesis (options), per utterance, with y_offsets = x_offsets."""
    import packed_common as pk
    Pa = pk.Packed(world, fs, n_samples, n, seed=31)
    c = Pa.c
    x, _ = Pa.x_packed()
    t, f0, sp, ap, fo = world.analyze_packed(pc.make(world, x), Pa.xo, fs, c.ao, **c.kw)
    scale, ratio = so.factors(n)
    world.modify_packed(f0, sp, fo, fs, c.sizes, f0_scale=scale, spectral_ratio=ratio)
    y = world.synthesis_packed(f0, sp, ap, fo, c.sizes, FP, fs, Pa.xo)
    X = pc.make(world, c.x)
    tb, fb, spb, apb, fl = world.analyze_batch(X, fs, c.ao, x_lengths=c.lens, **c.kw)
    fl = [int(v) for v in (fl.tolist() if hasattr(fl, "tolist") else fl)]
    world.modify(fb, spb, fs, c.sizes, f0_scale=scale, spectral_ratio=ratio, f0_lengths=fl)
    yb = world.synthesis(fb, spb, apb, c.sizes, FP, fs, max(c.lens), f0_lengths=fl, y_lengths=c.lens)
    world.synchronize()
    y, yb = pc.to_np(y), pc.to_np(yb)
    assert len(y) == Pa.xo[-1]
    for u in range(n):
        assert np.array_equal(y[Pa.xo[u]:Pa.xo[u + 1]], yb[u, :c.lens[u]]), f"round trip: utterance {u} differs"


def check_long_among_short(world, fs, long_s, short_s, n_short, budget):
    """One long utterance among many short ones at a budget that forces several passes: every sample equals the padded
    call's, in fewer passes (fewer launches) than the padded call at the same budget."""
    n = n_short + 1
    sizes = [so.sizes_of(world, fs, 2)[1]] * n
    fl_long, yl_long = int(1000.0 * long_s / FP) + 1, int(long_s * fs)
    fl_short, yl_short = int(1000.0 * short_s / FP) + 1, int(short_s * fs)
    lens = [(fl_short, yl_short)] * n
    lens[n // 3] = (fl_long, yl_long)
    P = Packed(world, fs, sizes, long_s, dims=24, seed=7, lens=lens)
    small = _with_budget(world, budget)
    try:
        before = small.launch_count()
        want = run_padded(world, P, "coded", budget_world=small)
        padded = small.launch_count() - before
        before = small.launch_count()
        got, clean = run_packed(small, P, "coded")
        packed = small.launch_count() - before
    finally:
        small.close()
    assert clean
    assert_equal(P, got, want, "long among short")
    assert packed < padded, f"launches: packed {packed}, padded {padded}: the packed call took no fewer passes"


def check_relaid(world, fs=16000, n=4, seconds=0.3):
    """One utterance at 2 kHz takes the relaid pass (one more time-base launch) and still equals the padded call."""
    sizes = sizes_at(world, fs, n)
    P = Packed(world, fs, sizes, seconds, seed=5, high=1)
    low = Packed(world, fs, sizes, seconds, seed=5)
    counts = []
    for Q in (P, low):
        before = world.launch_count()
        run_packed(world, Q, "coded")
        counts.append(world.launch_count() - before)
    assert counts[0] > counts[1], f"launches {counts}: the 2 kHz utterance did not take the relaid pass"
    got, clean = run_packed(world, P, "coded")
    assert clean
    assert_equal(P, got, run_padded(world, P, "coded"), "relaid pass")


def check_edges(world, fs=16000):
    """Utterances of 2 frames and 2 samples among longer ones, one utterance alone, and none."""
    sizes = sizes_at(world, fs, 4)
    lens = [(2, 2), (61, 4800), (2, 2), (30, 2400)]
    P = Packed(world, fs, sizes, 0.3, lens=lens)
    for family in ("full", "pcm16"):
        got, clean = run_packed(world, P, family)
        assert clean
        want = run_padded(world, P, family)
        for u in range(P.n):
            assert np.array_equal(P.seg(got, u), want[u, :P.b.y_len[u]]), f"{family}: utterance {u} differs"
    one = Packed(world, fs, sizes[:1], 0.2)
    got, clean = run_packed(world, one, "coded")
    assert clean
    assert_equal(one, got, run_padded(world, one, "coded"), "one utterance")
    before = world.launch_count()
    y = world.synthesis_packed(pc.make(world, np.zeros(1)), pc.make(world, np.zeros((1, 3))),
                               pc.make(world, np.zeros((1, 3))), [0], [], FP, fs, [0])
    world.modify_packed(pc.make(world, np.zeros(1)), pc.make(world, np.zeros((1, 3))), [0], fs, [], f0_scale=[])
    world.synchronize()
    assert len(y) == 0 and world.launch_count() == before, "an empty batch queued work"


def check_vs_ref(world, ref, fs=16000, n=3, seconds=0.3):
    """A few utterances of synthesis_packed within the reference's tolerance of its own Synthesis."""
    P = Packed(world, fs, sizes_at(world, fs, n), seconds, seed=17)
    got, _ = run_packed(world, P, "full")
    for u in range(P.n):
        a, z, bins = P.fo[u], P.fo[u + 1], P.b.sizes[u] // 2 + 1
        yr = ref.synthesis(P.f0[a:z], np.ascontiguousarray(P.sp[a:z, :bins]), np.ascontiguousarray(P.ap[a:z, :bins]),
                           P.b.sizes[u], FP, fs, P.b.y_len[u])
        e = np.abs(P.seg(got, u) - yr).max() / max(np.abs(yr).max(), 1e-300)
        assert e <= 1e-9, f"utterance {u} (fft_size {P.b.sizes[u]}): {e:.2e} of the peak"


def off_arg(v):
    v = [int(t) for t in v]
    return (C.c_longlong * len(v))(*v)


def pc_ptr(a):
    if a is None:
        return None
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def check_invalid(world, fs=16000):
    """Every bad argument is EINVAL before anything is queued: no launch, outputs untouched, last_error naming the bad
    utterance k."""
    n, k = 4, 2
    sizes = sizes_at(world, fs, n)
    P = Packed(world, fs, sizes, 0.1, seed=13)
    lib = world.lib
    F, SP, AP = pc.make(world, P.f0), pc.make(world, P.sp), pc.make(world, P.ap)
    CSP, CAP = pc.make(world, P.csp), pc.make(world, P.cap)
    y = pc.make(world, np.full(P.Y, -7.0))
    host_y = np.full(P.Y, -7.0)
    fo, yo = list(P.fo), list(P.yo)

    def bad(v, at, val):
        out = list(v)
        out[at] = val
        return out

    def moved(v, at, by):   # utterance `at` shorter or longer by `by`, the others as they were
        out = list(v)
        for i in range(at + 1, len(out)):
            out[i] += by
        return out

    calls = {
        "full": lambda s=sizes, f=fo, yy=yo, row=P.width: lib.world_b200_synthesis_packed(
            world._h, pc_ptr(F), n, off_arg(f), pc_ptr(SP), pc_ptr(AP), row, None if s is None else (C.c_int * n)(*s),
            FP, fs, off_arg(yy), pc_ptr(y)),
        "coded": lambda s=sizes, f=fo, yy=yo, row=None: lib.world_b200_synthesis_coded_packed(
            world._h, pc_ptr(F), n, off_arg(f), pc_ptr(CSP), 24, pc_ptr(CAP),
            None if s is None else (C.c_int * n)(*s), FP, fs, off_arg(yy), None, None, 0, pc_ptr(y)),
        "host": lambda s=sizes, f=fo, yy=yo, row=None: lib.world_b200_synthesis_coded_host_packed(
            world._h, P.f0.ctypes.data, n, off_arg(f), P.csp.ctypes.data, 24, P.cap.ctypes.data,
            None if s is None else (C.c_int * n)(*s), FP, fs, off_arg(yy), None, None, 0, host_y.ctypes.data),
        "modify": lambda s=sizes, f=fo, yy=None, row=P.width: lib.world_b200_modify_packed(
            world._h, pc_ptr(F), n, off_arg(f), pc_ptr(SP), row, None if s is None else (C.c_int * n)(*s), fs, None,
            (C.c_double * n)(*[0.9] * n)),
    }
    syn = ("full", "coded", "host")
    cases = [(fam, "fft_sizes NULL", dict(s=None), "fft_sizes must be given") for fam in calls]
    cases += [(fam, "fft_size 1000", dict(s=bad(sizes, k, 1000)), f"utterance {k})") for fam in calls]
    cases += [(fam, "f_offsets[0] = 1", dict(f=bad(fo, 0, 1)), "f_offsets[0] = 1") for fam in calls]
    cases += [(fam, "y_offsets[0] = 1", dict(yy=bad(yo, 0, 1)), "y_offsets[0] = 1") for fam in syn]
    cases += [(fam, "one frame", dict(f=moved(fo, k, 1 - (fo[k + 1] - fo[k]))), f"utterance {k})") for fam in syn]
    cases += [(fam, "one sample", dict(yy=moved(yo, k, 1 - (yo[k + 1] - yo[k]))), f"utterance {k})") for fam in syn]
    cases += [(fam, "descending f_offsets", dict(f=moved(fo, k, -(fo[k + 1] - fo[k]) - 1)), f"utterance {k})")
              for fam in calls]
    cases += [(fam, "2^31 samples", dict(yy=moved(yo, k, 2 ** 31)), f"utterance {k})") for fam in syn]
    cases += [(fam, "row_stride below a size's bins", dict(row=sizes[k] // 2), f"utterance {k})")
              for fam in ("full", "modify")]
    sp0 = pc.to_np(SP).copy()
    for fam, what, kw, named in cases:
        before = world.launch_count()
        rc = calls[fam](**kw)
        err = lib.world_b200_last_error(world._h).decode()
        assert rc == so.EINVAL, f"{fam}, {what}: returned {rc}"
        assert world.launch_count() == before, f"{fam}, {what}: kernels were launched"
        assert (pc.to_np(y) == -7.0).all() and (host_y == -7.0).all(), f"{fam}, {what}: the output was written"
        assert np.array_equal(pc.to_np(SP), sp0), f"{fam}, {what}: the rows were changed"
        assert named in err, f"{fam}, {what}: last_error {err!r} does not name {named!r}"
    with pytest.raises(ValueError):
        world.synthesis_packed(F, SP, AP, fo, sizes, FP, fs, yo[:-1])   # offsets of different counts
    before = world.launch_count()
    assert calls["coded"]() == 0
    world.synchronize()
    assert world.launch_count() > before and not (pc.to_np(y) == -7.0).all()
