"""Checks of Synthesis, modification and the voice transform with one fft_size per utterance
(world_b200_synthesis_batch_options, world_b200_synthesis_coded_batch_options, world_b200_synthesis_coded_host_options,
world_b200_modify_batch_options, world_b200_transform_*_spectral_options); the same assertions run against the host
emulation (CPU) and the CUDA library (-m gpu).

The oracle is the one-size call of the same family on each utterance alone at its own size: every row of a mixed call
must equal it bit for bit, whatever the order of the sizes, the scratch budget, or a relaid pass."""
import ctypes as C

import numpy as np

import test_parity_common as pc
from test_stage_paths import SMALL_BUDGET, _with_budget

EINVAL = 3
FP = 5.0
# per-speaker F0 floors -> CheapTrick sizes: 150 / 71 / 40 Hz give 512 / 1024 / 2048 at 16 kHz; 71 / 40 Hz give 2048 /
# 4096 at 48 kHz
FLOORS = {16000: (150.0, 71.0, 40.0), 48000: (71.0, 40.0)}


def ct_options(world, fs, floors):
    """The reference's recipe: the option's f0_floor set to the speaker's floor, fft_size derived from it."""
    out = []
    for lo in floors:
        o = world.cheaptrick_option(fs)
        o.f0_floor = lo
        o.fft_size = world.lib.GetFFTSizeForCheapTrick(fs, C.byref(o))
        out.append(o)
    return out


def sizes_of(world, fs, n):
    """n sizes from the rate's floors, interleaved (not grouped): floor u % k for utterance u."""
    floors = FLOORS[fs]
    return [o.fft_size for o in ct_options(world, fs, [floors[u % len(floors)] for u in range(n)])]


class Batch:
    """A ragged mixed batch: f0, full rows (row_stride = the largest bins + 3) and the same envelopes coded at each
    utterance's own size, as host arrays.  high: the utterance whose f0 is 2 kHz, above the 1,200 pulses per second a
    pass is first laid out for, so that its pass is laid out again."""

    def __init__(self, world, fs, sizes, seconds, dims, seed=0, high=None):
        rng = np.random.default_rng(seed)
        n = len(sizes)
        self.fs, self.sizes, self.dims, self.n = fs, list(sizes), dims, n
        ns = int(seconds * fs)
        self.y_len = [ns - (u * ns) // (2 * n + 1) for u in range(n)]
        self.f_len = [int(1000.0 * m / fs / FP) + 1 - (u % 3) for u, m in enumerate(self.y_len)]
        L = max(self.f_len)
        self.row = max(sizes) // 2 + 1 + 3
        self.f0 = np.zeros((n, L))
        self.sp = np.full((n, L, self.row), 7.0)    # padding values: never read
        self.ap = np.full((n, L, self.row), 0.5)
        n_ap = max(1, world.number_of_aperiodicities(fs))
        self.csp = np.zeros((n, L, dims))
        self.cap = np.zeros((n, L, n_ap))
        for u, f in enumerate(sizes):
            m, bins = self.f_len[u], f // 2 + 1
            k = np.arange(bins) / bins
            voiced = rng.uniform(size=m) < 0.85
            self.f0[u, :m] = np.where(voiced, rng.uniform(90.0, 300.0) * (1 + 0.2 * np.sin(np.arange(m) / 30.0)), 0.0)
            if u == high:
                self.f0[u, :m] = 2000.0
            sp = np.exp(-6.0 * k[None, :] + 0.3 * rng.normal(size=(m, 1))) * 1e-3
            ap = np.clip(k[None, :] ** 2 + 0.05 * rng.uniform(size=(m, bins)), 1e-3, 1 - 1e-12)
            self.sp[u, :m, :bins] = sp
            self.ap[u, :m, :bins] = ap
            self.csp[u, :m] = pc.to_np(world.code_spectral_envelope(pc.make(world, sp[None]), fs, f, dims))[0]
            if world.number_of_aperiodicities(fs) > 0:
                self.cap[u, :m] = pc.to_np(world.code_aperiodicity(pc.make(world, ap[None]), fs, f))[0]
        world.synchronize()
        self.Y = max(self.y_len)

    def one(self, u):
        """Utterance u alone: (f0, full sp, full ap at its own bins, coded sp, coded ap), host arrays."""
        bins = self.sizes[u] // 2 + 1
        m = self.f_len[u]
        return (self.f0[u:u + 1, :m], self.sp[u:u + 1, :m, :bins], self.ap[u:u + 1, :m, :bins],
                self.csp[u:u + 1, :m], self.cap[u:u + 1, :m])


def factors(n):
    return [1.0 + 0.1 * (u % 3) - 0.05 for u in range(n)], [0.85 + 0.1 * (u % 4) for u in range(n)]


def run_family(world, b, family, sizes=None, budget_world=None):
    """The mixed call of one family on b (sizes: per-utterance list, or one int for every utterance): host rows out."""
    w = budget_world or world
    sizes = b.sizes if sizes is None else sizes
    F = pc.make(w, b.f0)
    fs = b.fs
    scale, ratio = factors(b.n)
    if family == "full":
        y = w.synthesis(F, pc.make(w, b.sp), pc.make(w, b.ap), sizes, FP, fs, b.Y, f0_lengths=b.f_len,
                        y_lengths=b.y_len)
    elif family == "modify":
        f0, sp = pc.make(w, b.f0.copy()), pc.make(w, b.sp.copy())   # in place: never on the batch's own rows
        w.modify(f0, sp, fs, sizes, f0_scale=scale, spectral_ratio=ratio, f0_lengths=b.f_len)
        w.synchronize()
        return pc.to_np(f0), pc.to_np(sp)
    elif family == "host":
        y = w.synthesis_coded_host(b.f0, b.csp, b.cap, sizes, FP, fs, b.Y, nbit=16, f0_lengths=b.f_len,
                                   y_lengths=b.y_len, f0_scale=scale, spectral_ratio=ratio)
    else:
        kw = {}
        if family == "pcm16":
            kw["dtype"] = "int16"
        if family == "modified":
            kw.update(f0_scale=scale, spectral_ratio=ratio)
        y = w.synthesis_coded(F, pc.make(w, b.csp), pc.make(w, b.cap), sizes, FP, fs, b.Y, f0_lengths=b.f_len,
                              y_lengths=b.y_len, **kw)
    w.synchronize()
    return pc.to_np(y)


def run_one(world, b, family, u):
    """The one-size call of the family on utterance u alone at its size."""
    f0, sp, ap, csp, cap = b.one(u)
    fs, f, yl = b.fs, b.sizes[u], b.y_len[u]
    scale, ratio = factors(b.n)
    if family == "full":
        y = world.synthesis(pc.make(world, f0), pc.make(world, sp), pc.make(world, ap), f, FP, fs, yl)
    elif family == "modify":
        F, S = pc.make(world, f0.copy()), pc.make(world, sp.copy())
        world.modify(F, S, fs, f, f0_scale=[scale[u]], spectral_ratio=[ratio[u]])
        world.synchronize()
        return pc.to_np(F), pc.to_np(S)
    elif family == "host":
        y = world.synthesis_coded_host(f0, csp, cap, f, FP, fs, yl, nbit=16, f0_scale=[scale[u]],
                                       spectral_ratio=[ratio[u]])
    else:
        kw = {}
        if family == "pcm16":
            kw["dtype"] = "int16"
        if family == "modified":
            kw.update(f0_scale=[scale[u]], spectral_ratio=[ratio[u]])
        y = world.synthesis_coded(pc.make(world, f0), pc.make(world, csp), pc.make(world, cap), f, FP, fs, yl, **kw)
    world.synchronize()
    return pc.to_np(y)


FAMILIES = ("full", "coded", "pcm16", "modified", "host", "modify")


def check_rows(world, b, family, got):
    """Every row of the mixed call equals the one-size call on that utterance alone, bit for bit."""
    for u in range(b.n):
        want = run_one(world, b, family, u)
        if family == "modify":
            m, bins = b.f_len[u], b.sizes[u] // 2 + 1
            assert np.array_equal(got[0][u, :m], want[0][0]), f"modify: f0 of utterance {u} differs"
            assert np.array_equal(got[1][u, :m, :bins], want[1][0]), f"modify: envelope of utterance {u} differs"
            assert (got[1][u, :m, bins:] == 7.0).all(), f"modify: padding of utterance {u} was written"
            continue
        yl = b.y_len[u]
        assert np.array_equal(got[u, :yl], want[0]), f"{family}: utterance {u} (fft_size {b.sizes[u]}) differs"
        assert np.abs(got[u, :yl]).max() > 0, f"{family}: utterance {u} is silent"


def check_family(world, fs, family, n=5, seconds=0.3, dims=24, seed=1, high=None):
    b = Batch(world, fs, sizes_of(world, fs, n), seconds, dims, seed=seed, high=high)
    assert len(set(b.sizes)) > 1
    check_rows(world, b, family, run_family(world, b, family))
    return b


def check_relaid(world, fs, n=4, seconds=0.3, dims=24):
    """One utterance at 2 kHz forces its pass to be laid out again (one more time-base launch); every row still equals
    its one-size call."""
    sizes = sizes_of(world, fs, n)
    b = Batch(world, fs, sizes, seconds, dims, seed=5, high=1)
    low = Batch(world, fs, sizes, seconds, dims, seed=5)
    counts = []
    for bb in (b, low):
        before = world.launch_count()
        got = run_family(world, bb, "coded")
        counts.append(world.launch_count() - before)
    assert counts[0] == counts[1] + 1, f"launches {counts}: the 2 kHz utterance did not take the relaid pass"
    check_rows(world, b, "coded", run_family(world, b, "coded"))


def check_all_equal(world, fs=16000, n=3, seconds=0.3, dims=24):
    """Sizes all equal: the options call equals the existing call (rows of exactly that size's bins)."""
    f = sizes_of(world, fs, 2)[1]
    b = Batch(world, fs, [f] * n, seconds, dims, seed=9)
    bins = f // 2 + 1
    F = pc.make(world, b.f0)
    sp, ap = np.ascontiguousarray(b.sp[:, :, :bins]), np.ascontiguousarray(b.ap[:, :, :bins])
    y_old = world.synthesis(F, pc.make(world, sp), pc.make(world, ap), f, FP, fs, b.Y, f0_lengths=b.f_len,
                            y_lengths=b.y_len)
    y_new = world.synthesis(F, pc.make(world, sp), pc.make(world, ap), [f] * n, FP, fs, b.Y, f0_lengths=b.f_len,
                            y_lengths=b.y_len)
    world.synchronize()
    assert np.array_equal(pc.to_np(y_old), pc.to_np(y_new))
    for family in ("coded", "pcm16", "modified"):
        assert np.array_equal(run_family(world, b, family, sizes=f), run_family(world, b, family)), family


def check_small_budget(world, fs=16000, n=6, seconds=2.0, dims=24):
    """At the smallest scratch budget the mixed call runs in several passes and gives the same rows."""
    b = Batch(world, fs, sizes_of(world, fs, n), seconds, dims, seed=11)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs, launches = [], []
        for w in (world, small):
            before = w.launch_count()
            outs.append(run_family(world, b, "modified", budget_world=w))
            launches.append(w.launch_count() - before)
    finally:
        small.close()
    assert launches[1] > launches[0], f"launches {launches}: the small budget did not cut the batch into passes"
    assert np.array_equal(outs[0], outs[1])


# ---- the transform ----------------------------------------------------------------------------------------------------
def transform_inputs(world, fs, n, seconds):
    from synth import synth_batch
    ns = int(seconds * fs)
    x = synth_batch([401 + u for u in range(n)], fs, ns).numpy()
    lens = [ns - (u * ns) // 9 for u in range(n)]
    for u, m in enumerate(lens):
        x[u, m:] = 0.0
    floors = FLOORS[fs]
    cts = ct_options(world, fs, [floors[u % len(floors)] for u in range(n)])
    return x, lens, cts


def check_transform(world, fs=16000, n=4, seconds=0.4, host=False):
    """transform with per-utterance CheapTrick options equals, row by row, the one-option transform of each utterance
    alone with its option (pitch, formant and tempo factors per utterance)."""
    from world_b200.api import F0_DIO_STONEMASK
    x, lens, cts = transform_inputs(world, fs, n, seconds)
    ao = world.analysis_option(fs, F0_DIO_STONEMASK)
    scale, ratio = factors(n)
    ts = [(1.0, 1.25, 0.8)[u % 3] for u in range(n)]
    call = world.transform_host if host else world.transform
    X = x if host else pc.make(world, x)
    y, yl = call(X, 0, fs, ao, f0_scale=scale, spectral_ratio=ratio, time_scale=ts, x_lengths=lens,
                 cheaptrick_options=cts)
    world.synchronize()
    y = pc.to_np(y)
    for u in range(n):
        ao1 = world.analysis_option(fs, F0_DIO_STONEMASK)
        C.memmove(C.byref(ao1.cheaptrick), C.byref(cts[u]), C.sizeof(cts[u]))
        xu = np.ascontiguousarray(x[u:u + 1, :lens[u]])
        y1, yl1 = call(xu if host else pc.make(world, xu), 0, fs, ao1, f0_scale=[scale[u]], spectral_ratio=[ratio[u]],
                       time_scale=[ts[u]])
        world.synchronize()
        assert yl1[0] == yl[u]
        assert np.array_equal(y[u, :yl[u]], pc.to_np(y1)[0]), f"transform: utterance {u} differs"
    return x, lens, cts, y, yl


def check_transform_stepwise(world, fs=16000, n=4, seconds=0.4):
    """transform_batch_spectral_options equals the stepwise chain: DIO + StoneMask (analyze_coded_batch's F0 rows),
    cheaptrick / d4c with per-utterance options -> modify_batch_options -> synthesis_batch_options, bit for bit."""
    from world_b200.api import F0_DIO_STONEMASK
    x, lens, cts = transform_inputs(world, fs, n, seconds)
    ao = world.analysis_option(fs, F0_DIO_STONEMASK)
    scale, ratio = factors(n)
    X = pc.make(world, x)
    y, yl = world.transform(X, 0, fs, ao, f0_scale=scale, spectral_ratio=ratio, x_lengths=lens, cheaptrick_options=cts)
    t, f0, _, _, fl = world.analyze_coded_batch(X, 0, fs, ao, 8, x_lengths=lens)
    sizes = [o.fft_size for o in cts]
    sp = world.cheaptrick(X, fs, t, f0, cts, x_lengths=lens, f0_lengths=fl)
    ap = world.d4c(X, fs, t, f0, sizes, x_lengths=lens, f0_lengths=fl)
    world.modify(f0, sp, fs, sizes, f0_scale=scale, spectral_ratio=ratio, f0_lengths=fl)
    want = world.synthesis(f0, sp, ap, sizes, ao.dio.frame_period, fs, max(yl), f0_lengths=fl, y_lengths=yl)
    world.synchronize()
    assert np.array_equal(pc.to_np(y), pc.to_np(want))


# ---- rejections -------------------------------------------------------------------------------------------------------
def check_invalid(world, fs=16000):
    """Every bad argument is EINVAL before anything is queued: no launch, outputs untouched, last_error naming the bad
    utterance k; the context works afterwards."""
    n, k = 4, 2
    sizes = sizes_of(world, fs, n)
    b = Batch(world, fs, sizes, 0.1, 24, seed=13)
    lib = world.lib
    F, SP, AP = pc.make(world, b.f0), pc.make(world, b.sp), pc.make(world, b.ap)
    CSP, CAP = pc.make(world, b.csp), pc.make(world, b.cap)
    y = pc.make(world, np.full((n, b.Y), -7.0))
    L = b.f0.shape[1]
    fl, yl = (C.c_int * n)(*b.f_len), (C.c_int * n)(*b.y_len)
    ptr = pc_ptr

    def arr(v):
        return None if v is None else (C.c_int * n)(*v)

    def bad(at, v):
        out = list(sizes)
        out[at] = v
        return out

    calls = {
        "full": lambda s=sizes, row=b.row: lib.world_b200_synthesis_batch_options(
            world._h, ptr(F), fl, n, L, ptr(SP), ptr(AP), row, arr(s), FP, fs, yl, b.Y, ptr(y)),
        "coded": lambda s=sizes, dims=24: lib.world_b200_synthesis_coded_batch_options(
            world._h, ptr(F), fl, n, L, ptr(CSP), dims, ptr(CAP), arr(s), FP, fs, yl, b.Y, None, None, 0, ptr(y)),
        "host": lambda s=sizes, dims=24: lib.world_b200_synthesis_coded_host_options(
            world._h, b.f0.ctypes.data, fl, n, L, b.csp.ctypes.data, dims, b.cap.ctypes.data, arr(s), FP, fs, yl,
            b.Y, None, None, 0, host_y.ctypes.data),
        "modify": lambda s=sizes, row=b.row: lib.world_b200_modify_batch_options(
            world._h, ptr(F), fl, n, L, ptr(SP), row, arr(s), fs, None, (C.c_double * n)(*[0.9] * n)),
    }
    host_y = np.full((n, b.Y), -7.0)
    small_first = sizes.index(min(sizes))
    cases = [(fam, "fft_sizes NULL", dict(s=None), "fft_sizes must be given") for fam in calls]
    cases += [(fam, "fft_size 1000", dict(s=bad(k, 1000)), f"utterance {k}") for fam in calls]
    cases += [(fam, "fft_size 8192", dict(s=bad(k, 8192)), f"utterance {k}") for fam in ("full", "coded", "host")]
    cases += [(fam, "row_stride below a size's bins", dict(row=sizes[k] // 2), f"utterance {k}")
              for fam in ("full", "modify")]
    # number_of_dimensions above the smallest size's half (the first utterance of that size is named)
    cases += [(fam, "dims > fft_size/2", dict(dims=min(sizes) // 2 + 1), f"utterance {small_first}")
              for fam in ("coded", "host")]
    sp0 = pc.to_np(SP).copy()
    for fam, what, kw, named in cases:
        before = world.launch_count()
        rc = calls[fam](**kw)
        err = lib.world_b200_last_error(world._h).decode()
        assert rc == EINVAL, f"{fam}, {what}: returned {rc}"
        assert world.launch_count() == before, f"{fam}, {what}: kernels were launched"
        assert (pc.to_np(y) == -7.0).all() and (host_y == -7.0).all(), f"{fam}, {what}: the output was written"
        assert np.array_equal(pc.to_np(SP), sp0), f"{fam}, {what}: the rows were changed"
        assert named in err, f"{fam}, {what}: last_error {err!r} does not name {named!r}"
    before = world.launch_count()
    assert calls["coded"]() == 0
    world.synchronize()
    assert world.launch_count() > before and not (pc.to_np(y) == -7.0).all()


def pc_ptr(a):
    if a is None:
        return None
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data
