"""Synthesis on caller-built f0, envelope and aperiodicity rows: constructed tables aimed at the guards and thresholds
of the time base and of the pulse responses, at every rate, through three call forms that must agree bit for bit (the
lone padded call of each utterance, the per-utterance _options call of the whole batch, and the _packed call) and
compared sample by sample with the reference.  The same assertions run against the host emulation (CPU) and the CUDA
library (-m gpu).

Each builder below cites the line of the reference's synthesis.cpp (codec.cpp for the coded rows) it is aimed at, and
the kernel line of wb_synthesis.cu / wb_codec.cu that restates it.  Where a builder needs a pulse at a particular
place (on a frame, on the V/UV midpoint), it finds it with `timebase`, a numpy restatement of the reference's time
base in the reference's operation order, and asserts that the table reaches it.

The bound: where the reference sample yr[s] is finite, |y[s] - yr[s]| <= 1e-9 max|yr| over [s - fft/2, s + fft/2],
the span of every response that covers s.  The peak is local, so a flipped decision in a quiet stretch cannot hide
under a loud one.  Where yr[s] is NaN, y[s] must be NaN too.

Every case keeps each pulse's noise_size (the distance to the next pulse) at most fft_size: the reference writes that
many noise samples into an fft_size buffer, so beyond it the reference is not defined (fft_sizes_common.py)."""
import numpy as np

import test_parity_common as pc

RATES = [8000, 11025, 16000, 22050, 24000, 44100, 48000]
SIZES = [1 << k for k in range(4, 13)]                # 16 ... 4096, every size Synthesis takes
FPS = [1.0, 2.5, 5.0, 10.0, 4.3]                       # ms; 4.3 ms puts frames off the sample grid at every rate
REL = 1e-9
SAFE = 1.0 - 1e-12                                     # kMySafeGuardMinimum's complement: GetSafeAperiodicity's top

# worst local error per family (printed by report(); pytest -s shows them)
STATS = {}


def _note(key, value):
    STATS[key] = max(STATS.get(key, 0.0), float(value))


def report():
    for k in sorted(STATS):
        print(f"synthesis edges: {k}: {STATS[k]:.3g}")


def up(v):
    return float(np.nextafter(v, np.inf))


def down(v):
    return float(np.nextafter(v, -np.inf))


def default_fft(fs):
    """CheapTrick's default fft_size at fs (the size analysis output comes at)"""
    return 1 << int(np.ceil(np.log2(3.0 * fs / 71.0 + 1)))


def lowest_f0(fs, fft):
    return fs // fft + 1.0                             # synthesis.cpp:361: integer division, then + 1.0


class Case:
    """One utterance: f0 [L], envelope and aperiodicity rows [L, fft/2 + 1], y_length samples, frame period in ms."""

    def __init__(self, name, fs, fft, fp, f0, sp, ap, y_len):
        self.name, self.fs, self.fft, self.fp = name, fs, fft, fp
        self.f0 = np.ascontiguousarray(f0, dtype=np.float64)
        self.sp = np.ascontiguousarray(sp, dtype=np.float64)
        self.ap = np.ascontiguousarray(ap, dtype=np.float64)
        self.y_len = int(y_len)
        L, bins = len(self.f0), fft // 2 + 1
        assert L >= 2 and self.sp.shape == (L, bins) and self.ap.shape == (L, bins) and self.y_len >= 2, name
        tb = timebase(self.f0, fs, fft, fp, self.y_len)
        gaps = np.diff(tb.idx)
        assert not len(gaps) or gaps.max() <= fft, f"{name}: noise_size {gaps.max()} > fft_size {fft}"
        self.tb = tb


def envelope(rng, fs, fft, L, scale=1e-3):
    """A smooth positive envelope per frame, a little different from frame to frame."""
    k = np.arange(fft // 2 + 1) / (fft // 2 + 1)
    tilt = rng.uniform(3.0, 6.0, size=(L, 1))
    ripple = 0.4 * np.sin(2 * np.pi * (k[None, :] * rng.uniform(2, 6, size=(L, 1)) + rng.uniform(size=(L, 1))))
    return scale * np.exp(-tilt * k[None, :] + ripple)


def aperiodicity(rng, fft, L, lo=0.002, hi=0.95):
    """Aperiodicity rising with frequency, between lo and hi."""
    k = np.arange(fft // 2 + 1) / (fft // 2 + 1)
    return np.clip(lo + (hi - lo) * k[None, :] ** 1.5 * rng.uniform(0.7, 1.0, size=(L, 1))
                   + 0.02 * rng.uniform(size=(L, fft // 2 + 1)), lo, hi)


# ------------------------------------------------------------------------------------------------------------ time base
class TimeBase:
    pass


def timebase(f0, fs, fft, fp_ms, y_len):
    """GetTimeBase (synthesis.cpp:288-321) in numpy, in the reference's operation order: the coarse arrays with the
    extrapolated end point (:231-240), histc's segment (the first node above t, at most L), interp1, the > 0.5 decision
    (:305), 500 Hz in unvoiced samples, the index-order phase sum (np.cumsum adds in index order), fmod and the
    |wrap[i+1] - wrap[i]| > pi test (:260).  Returns the pulse indices, the raw interpolated vuv, and for each pulse
    whether it falls on a frame (GetSpectralEnvelope's floor == ceil, :144-150)."""
    fp = fp_ms / 1000.0
    L = len(f0)
    low = lowest_f0(fs, fft)
    with np.errstate(invalid="ignore"):
        cf = np.where(f0 < low, 0.0, f0)
        cv = np.where(cf == 0.0, 0.0, 1.0)
        cf = np.append(cf, cf[-1] * 2 - cf[-2])
        cv = np.append(cv, cv[-1] * 2 - cv[-2])
        ct = np.arange(L + 1) * fp
        t = np.arange(y_len) / float(fs)
        k = np.clip(np.searchsorted(ct, t, side="right"), 1, L)
        s = (t - ct[k - 1]) / (ct[k] - ct[k - 1])
        fi = cf[k - 1] + s * (cf[k] - cf[k - 1])
        vi = cv[k - 1] + s * (cv[k] - cv[k - 1])
        v = vi > 0.5
        phase = np.cumsum(2.0 * np.pi * np.where(v, fi, 500.0) / fs)
        wrap = np.fmod(phase, 2.0 * np.pi)
        idx = np.flatnonzero(np.abs(np.diff(wrap)) > np.pi)
    tb = TimeBase()
    tb.idx, tb.vi, tb.voiced = idx, vi, v
    ct_p = idx / float(fs)
    fl = np.minimum(L - 1, np.floor(ct_p / fp).astype(np.int64))
    ce = np.minimum(L - 1, np.ceil(ct_p / fp).astype(np.int64))
    tb.exact = fl == ce
    tb.fl, tb.ce = fl, ce
    return tb


# ------------------------------------------------------------------------------------------------------------- checking
def local_peak(yr, fft):
    """max |yr| over [s - fft/2, s + fft/2] for every s (NaN samples count as 0)"""
    from scipy.ndimage import maximum_filter1d
    a = np.where(np.isfinite(yr), np.abs(yr), 0.0)
    return maximum_filter1d(a, size=2 * (fft // 2) + 1, mode="constant", cval=0.0)


def local_error(y, yr, fft, what):
    """The bound of the module docstring; returns the worst |y - yr| / local peak over the finite samples."""
    y, yr = np.asarray(y), np.asarray(yr)
    nan_r = np.isnan(yr)
    bad = np.flatnonzero(np.isnan(y) != nan_r)
    assert bad.size == 0, f"{what}: NaN masks differ at samples {bad[:6].tolist()} (reference NaN: {nan_r[bad[:6]]})"
    peak = local_peak(yr, fft)
    fin = ~nan_r
    err = np.abs(y[fin] - yr[fin])
    lim = REL * peak[fin]
    over = np.flatnonzero(~(err <= lim))
    if over.size:
        s = np.flatnonzero(fin)[over[0]]
        raise AssertionError(f"{what}: sample {s}: {y[s]!r} vs reference {yr[s]!r}, local peak {peak[s]:.3e} "
                             f"({over.size} samples beyond 1e-9 of the local peak)")
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(peak[fin] > 0, err / np.where(peak[fin] > 0, peak[fin], 1.0), 0.0)
    return float(r.max()) if r.size else 0.0


def assert_same(a, b, what):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    assert a.shape == b.shape, f"{what}: shapes {a.shape} {b.shape}"
    bad = np.flatnonzero(a.view(np.uint64) != b.view(np.uint64))
    assert bad.size == 0, f"{what}: differs at samples {bad[:6].tolist()}: {a[bad[:3]]} vs {b[bad[:3]]}"


def pcm16(y):
    """wavwrite's quantisation as the library's pcm16_of states it: (int)(y * 32767) toward zero, saturated by sign
    beyond the int16 range, NaN -> 0"""
    s = np.asarray(y, dtype=np.float64) * 32767
    out = np.zeros(s.shape, dtype=np.int16)
    fin = ~np.isnan(s)
    out[fin] = np.clip(np.trunc(np.clip(s[fin], -40000.0, 40000.0)), -32768, 32767).astype(np.int16)
    return out


def run_cases(world, ref, family, cases):
    """Every case alone, then each frame period's cases as one _options batch and one _packed batch (bit for bit the
    lone call's samples), then each against the reference.  Returns the worst local error."""
    worst = 0.0
    for fp in sorted({c.fp for c in cases}):
        group = [c for c in cases if c.fp == fp]
        fs = group[0].fs
        assert all(c.fs == fs for c in group)
        W = max(c.fft // 2 + 1 for c in group)
        n, Lm, Y = len(group), max(len(c.f0) for c in group), max(c.y_len for c in group)
        F = np.zeros((n, Lm)); S = np.ones((n, Lm, W)); A = np.ones((n, Lm, W))
        for u, c in enumerate(group):
            L, b = len(c.f0), c.fft // 2 + 1
            F[u, :L] = c.f0; S[u, :L, :b] = c.sp; A[u, :L, :b] = c.ap
        sizes = [c.fft for c in group]
        fl, yl = [len(c.f0) for c in group], [c.y_len for c in group]
        mk = lambda a: pc.make(world, a)
        batch = world.synthesis(mk(F), mk(S), mk(A), sizes, fp, fs, Y, f0_lengths=fl, y_lengths=yl)
        fo = np.concatenate([[0], np.cumsum(fl)]).astype(np.int64)
        yo = np.concatenate([[0], np.cumsum(yl)]).astype(np.int64)
        Sp = np.concatenate([np.pad(c.sp, ((0, 0), (0, W - c.sp.shape[1])), constant_values=1.0) for c in group])
        Ap = np.concatenate([np.pad(c.ap, ((0, 0), (0, W - c.ap.shape[1])), constant_values=1.0) for c in group])
        packed = world.synthesis_packed(mk(np.concatenate([c.f0 for c in group])), mk(Sp), mk(Ap), fo, sizes, fp, fs,
                                        yo)
        world.synchronize()
        batch, packed = pc.to_np(batch), pc.to_np(packed)
        for u, c in enumerate(group):
            what = f"{family} fs {fs} fp {fp} fft {c.fft} {c.name}"
            lone = pc.to_np(world.synthesis(mk(c.f0[None]), mk(c.sp[None]), mk(c.ap[None]), c.fft, fp, fs, c.y_len))[0]
            world.synchronize()
            assert_same(batch[u, :c.y_len], lone, what + ": _options vs lone call")
            assert_same(packed[yo[u]:yo[u + 1]], lone, what + ": _packed vs lone call")
            yr = ref.synthesis(c.f0, c.sp, c.ap, c.fft, fp, fs, c.y_len)
            worst = max(worst, local_error(lone, yr, c.fft, what))
    _note(f"{family} worst |y - yr| / local peak", worst)
    return worst


# ------------------------------------------------------------------------------------------------ A. the time base
def floor_cases(fs):
    """A1: the synthesis floor fs / fft_size + 1.0 with integer division (synthesis.cpp:361, coarse_f0 at :233;
    wb_synthesis.cu:90, :101).  At every size whose 500 Hz unvoiced pulses fit the size, runs of frames at the floor,
    one ulp either side, and (where fs % fft_size != 0) between the integer and the floating-point floor, each between
    voiced runs.  A frame below the floor is unvoiced (500 Hz pulses); one at or above is voiced at about one pulse per
    fft_size, so any flipped decision moves every later pulse."""
    out = []
    for s, fft in enumerate(SIZES):
        if fs / 500.0 > 0.8 * fft:
            continue
        rng = np.random.default_rng([fs, fft, 1])
        fp = FPS[s % len(FPS)]
        lo, hi = lowest_f0(fs, fft), fs / fft + 1.0
        values = [lo, down(lo), up(lo), hi]
        if hi > lo:
            values += [0.5 * (lo + hi), down(hi), lo + 0.25 * (hi - lo)]
        run = max(2, min(int(np.ceil(0.5 * fft / fs / (fp / 1000.0))), int(0.04 / (fp / 1000.0)) + 1))
        bg = max(2.0 * hi, 120.0)
        f0 = [bg] * run
        for v in values:
            f0 += [v] * run + [bg] * run
        f0 = np.array(f0)
        L = len(f0)
        y_len = int(L * fp / 1000.0 * fs)
        out.append(Case(f"floor run {run}", fs, fft, fp, f0, envelope(rng, fs, fft, L), aperiodicity(rng, fft, L),
                        y_len))
    return out


def endpoint_cases(fs):
    """A2: the extrapolated end point coarse_f0[L] = 2 f0[L-1] - f0[L-2], coarse_vuv[L] likewise (synthesis.cpp:236-240;
    wb_synthesis.cu:103-104, :115-116): all four voicing combinations of the last two frames, a steep fall (300 -> 100
    Hz: the extrapolated f0 crosses zero and goes negative while the voicing stays 1, so the phase runs backwards, fmod
    takes negative phases and pulses are found on the falling side), a steep rise, and f0_length 2; y_length from 2 to
    three times L fp fs."""
    fft = default_fft(fs)
    ends = {"VV": (200.0, 200.0), "UV": (0.0, 200.0), "VU": (200.0, 0.0), "UU": (0.0, 0.0),
            "fall": (300.0, 100.0), "rise": (100.0, 300.0)}
    out = []
    for j, (name, (a, b)) in enumerate(ends.items()):
        for L in (2, 5):
            fp = FPS[(j + L) % len(FPS)]
            span = L * fp / 1000.0 * fs
            rng = np.random.default_rng([fs, j, L, 2])
            f0 = np.concatenate([np.full(L - 2, 180.0), [a, b]])
            for y_len in (2, int(span) // 2 + 1, int(round(span)), int(1.5 * span), int(3 * span)):
                if y_len < 2:
                    continue
                out.append(Case(f"end {name} L {L} y {y_len}", fs, fft, fp, f0, envelope(rng, fs, fft, L),
                                aperiodicity(rng, fft, L), y_len))
    return out


def vuv_cases(fs):
    """A3: the V/UV decision interpolated_vuv > 0.5 (synthesis.cpp:305; wb_synthesis.cu:117-118).  Runs of voiced and
    unvoiced frames, single voiced frames in silence and single unvoiced frames in voice, at every frame period: where
    fp fs / 2 is an integer (16 kHz at 5 ms, 48 kHz at 2.5 ms, 8 kHz at 1 ms) a sample lands on the midpoint between
    two frames and its interpolated vuv is exactly 0.5 (asserted); at the others no sample does."""
    fft = default_fft(fs)
    out, halves = [], 0
    pattern = [1, 1, 1, 0, 0, 0, 1, 0, 1, 1, 0, 1, 0, 0, 1, 1, 1, 0, 0, 1, 0, 0, 0, 1, 1, 0, 1, 1, 1]
    for j, fp in enumerate(FPS):
        rng = np.random.default_rng([fs, j, 3])
        f0 = np.array(pattern, dtype=np.float64) * rng.uniform(150.0, 260.0, size=len(pattern))
        L = len(f0)
        c = Case(f"vuv pattern", fs, fft, fp, f0, envelope(rng, fs, fft, L), aperiodicity(rng, fft, L),
                 int(L * fp / 1000.0 * fs))
        halves += int((c.tb.vi == 0.5).sum())
        out.append(c)
    if fs in (8000, 16000, 48000):
        assert halves > 0, f"vuv fs {fs}: no sample's interpolated vuv is exactly 0.5"
    return out


def pulse_cases(fs):
    """A4: dense and sparse pulses (synthesis.cpp:251-279, noise_size :371-372; wb_synthesis.cu:126-164).  f0 at 0.45,
    0.5, 0.75 and 1.5 fs: a pulse on nearly every sample, noise_size 1 (zero noise once the mean is removed) and 0 (the
    last pulse), and more pulses than the 1,200 per second the scratch is first laid out for, so the call lays its
    chunk out again; small sizes, at most 0.2 s.  And f0 just above the floor, about one pulse per fft_size."""
    out = []
    for j, r in enumerate((0.45, 0.5, 0.75, 1.5)):
        fft = SIZES[j % 3]
        fp = FPS[j]
        n = int(min(0.2, 400 * fft / fs / 100) * fs) if fs > 20000 else int(0.2 * fs)
        n = min(n, int(0.2 * fs))
        L = int(n / fs / (fp / 1000.0)) + 2
        rng = np.random.default_rng([fs, j, 4])
        f0 = np.full(L, r * fs)
        f0[L // 2:] *= 1.0 + 1e-3 * np.arange(L - L // 2)
        out.append(Case(f"dense {r} fs", fs, fft, fp, f0, envelope(rng, fs, fft, L), aperiodicity(rng, fft, L), n))
    for j, fft in enumerate((256, 1024, 4096)):
        lo = lowest_f0(fs, fft)
        if fs / lo > fft:
            continue
        fp = FPS[(j + 1) % len(FPS)]
        L = int(4 * fft / fs / (fp / 1000.0)) + 3
        rng = np.random.default_rng([fs, fft, 5])
        f0 = np.full(L, up(lo)) * (1.0 + 0.01 * rng.uniform(size=L))
        out.append(Case(f"sparse", fs, fft, fp, f0, envelope(rng, fs, fft, L), aperiodicity(rng, fft, L),
                        int(L * fp / 1000.0 * fs)))
    return out


def nonfinite_cases(fs):
    """A5: a NaN, an inf and a -inf in the middle of a voiced stretch (synthesis.cpp:233-234: NaN and inf are not below
    the floor, so they stay voiced; -inf is).  The NaN and inf make the total phase NaN from their segment on, so no
    pulse follows; -inf is an unvoiced frame."""
    fft = default_fft(fs)
    out = []
    for j, bad in enumerate((np.nan, np.inf, -np.inf)):
        fp = FPS[j + 1]
        L = 24
        rng = np.random.default_rng([fs, j, 6])
        f0 = rng.uniform(150.0, 220.0, size=L)
        f0[L // 2] = bad
        c = Case(f"f0 {bad}", fs, fft, fp, f0, envelope(rng, fs, fft, L), aperiodicity(rng, fft, L),
                 int(L * fp / 1000.0 * fs))
        if not np.isneginf(bad):
            assert c.tb.idx.max() < (L // 2) * fp / 1000.0 * fs, f"f0 {bad}: a pulse after the non-finite frame"
        out.append(c)
    return out


# ------------------------------------------------------------------------------------------------- B. pulse responses
def aimed_f0(fs, fp, L, rng):
    """A voiced contour whose pulses drift across the frame grid, so that some fall on a frame (floor == ceil) and the
    rest between frames"""
    return rng.uniform(0.97, 1.03) * (fs / (fp / 1000.0 * fs / 3.0)) * (1.0 + 0.002 * np.sin(np.arange(L)))


def _need_both(c, what):
    assert c.tb.exact.any() and (~c.tb.exact).any(), f"{what}: pulses on frames {c.tb.exact.sum()}, between " \
                                                     f"{(~c.tb.exact).sum()}"


def ap_clamp_cases(fs):
    """B6: GetSafeAperiodicity's clamps max(0.001, min(1 - 1e-12, ap)) (common.h:111-113, applied at
    synthesis.cpp:172 for a pulse on a frame and at :175-178 on both frames before interpolating; wb_synthesis.cu:245,
    :250).  Each frame's bins cycle through -1, 0, 0.001 and one ulp either side, 0.5, 1 - 1e-12 and one ulp either
    side, 1 and 2, shifted by one bin from frame to frame, so that a pulse between frames interpolates pairs such as
    (-1, 0.5); bin 0 stays at 0.3 (the periodic part is kept).  Pulses fall both on and between frames (asserted)."""
    vals = np.array([-1.0, 0.0, down(0.001), 0.001, up(0.001), 0.5, down(SAFE), SAFE, up(SAFE), 1.0, 2.0])
    out = []
    for j, fp in enumerate((2.5, 5.0, 10.0)):
        fft = default_fft(fs) if j != 1 else max(SIZES[0], default_fft(fs) // 2)
        if fs / 500.0 > fft:
            fft = default_fft(fs)
        L = 30
        rng = np.random.default_rng([fs, j, 7])
        f0 = aimed_f0(fs, fp, L, rng)
        bins = fft // 2 + 1
        ap = np.empty((L, bins))
        for i in range(L):
            ap[i] = np.resize(np.roll(vals, i), bins)
        ap[:, 0] = 0.3
        c = Case("ap clamps", fs, fft, fp, f0, envelope(rng, fs, fft, L), ap, int(L * fp / 1000.0 * fs))
        _need_both(c, f"ap clamps fs {fs} fp {fp}")
        out.append(c)
    return out


def ap_threshold():
    """The smallest double x with x * x > 0.999 (pow(x, 2.0) is correctly rounded, as x * x is), by bisection over
    the doubles' bit patterns."""
    lo, hi = np.float64(0.99).view(np.int64), np.float64(1.0).view(np.int64)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        x = np.int64(mid).view(np.float64)
        if x * x > 0.999:
            hi = mid
        else:
            lo = mid
    x = float(np.int64(hi).view(np.float64))
    assert x * x > 0.999 and down(x) * down(x) <= 0.999
    return x


def ap_drop_cases(fs):
    """B7: the periodic part is dropped when aperiodic_ratio[0] = GetSafeAperiodicity(ap[0])^2 > 0.999
    (synthesis.cpp:111; wb_synthesis.cu:259).  Bin 0 of the frames cycles through x*, one ulp either side (x*: the
    smallest double whose square exceeds 0.999), 0.9997 and 0.9993 (between 0.999 and 0.9995 once squared: kept under
    one of the two thresholds, dropped under the other); pulses between frames interpolate neighbours of x*."""
    x = ap_threshold()
    vals = [x, down(x), up(x), float(np.sqrt(0.9997)), float(np.sqrt(0.9993)), down(down(x)), up(up(x))]
    out = []
    for j, fp in enumerate((2.5, 5.0, 4.3)):
        fft = default_fft(fs)
        L = 28
        rng = np.random.default_rng([fs, j, 8])
        f0 = aimed_f0(fs, fp, L, rng)
        ap = aperiodicity(rng, fft, L)
        ap[:, 0] = np.resize(vals, L)
        if j == 2:
            ap[:, 0] = np.resize([x, x, down(x), down(x)], L)
        c = Case("ap[0] threshold", fs, fft, fp, f0, envelope(rng, fs, fft, L), ap, int(L * fp / 1000.0 * fs))
        _need_both(c, f"ap drop fs {fs} fp {fp}")
        out.append(c)
    return out


def env_sign_cases(fs):
    """B8: the envelope's absolute value (synthesis.cpp:152 on a frame, :156-157 between frames; wb_synthesis.cu:247,
    :251): negative rows, and rows of opposite sign in neighbouring frames, where |a|(1 - s) + |b| s differs from
    |a (1 - s) + b s|."""
    out = []
    for j, fp in enumerate((2.5, 5.0, 10.0)):
        fft = default_fft(fs)
        L = 26
        rng = np.random.default_rng([fs, j, 9])
        f0 = aimed_f0(fs, fp, L, rng)
        sp = envelope(rng, fs, fft, L)
        if j == 0:
            sp = -sp                                               # every row negative
        else:
            sp[1::2] *= -1.0                                       # signs alternate frame by frame
            sp[:, ::3] *= -1.0                                     # and bin by bin
        c = Case("negative envelope" if j == 0 else "alternating signs", fs, fft, fp, f0, sp,
                 aperiodicity(rng, fft, L), int(L * fp / 1000.0 * fs))
        _need_both(c, f"env sign fs {fs} fp {fp}")
        out.append(c)
    return out


def env_extreme_cases(fs):
    """B9: zero and extreme envelopes.  A zero envelope: the periodic log adds kMySafeGuardMinimum (synthesis.cpp:117-
    119), but the aperiodic one takes log(0) = -inf (:48-52), so the reference's response is NaN, and so are the
    samples it covers; the library must give NaN at exactly those samples.  Zero rows in the middle and at the end
    (the last pulse, whose noise_size is 0, :371-372), zero bins in one frame, and envelopes of 1e-300 and 1e300."""
    fft = default_fft(fs)
    out = []
    for j, (name, fp) in enumerate((("zero rows", 5.0), ("zero last rows", 2.5), ("zero bins", 10.0),
                                    ("1e-300", 4.3), ("1e300", 1.0))):
        L = 20
        rng = np.random.default_rng([fs, j, 10])
        f0 = rng.uniform(140.0, 240.0, size=L)
        sp = envelope(rng, fs, fft, L)
        if name == "zero rows":
            sp[8:10] = 0.0
        elif name == "zero last rows":
            sp[-2:] = 0.0
        elif name == "zero bins":
            sp[12, 5:9] = 0.0
        elif name == "1e-300":
            sp = sp / sp.max() * 1e-300
        else:
            sp = sp / sp.max() * 1e300
        out.append(Case(name, fs, fft, fp, f0, sp, aperiodicity(rng, fft, L), int(L * fp / 1000.0 * fs)))
    return out


def unvoiced_cases(fs):
    """B10: pulses in unvoiced stretches take log(spectrum) alone (current_vuv == 0, synthesis.cpp:46-52;
    wb_synthesis.cu:303), whatever the aperiodicity; here it is far from 1 and varies across bins, as it does in a
    caller's predicted rows (analysis puts 1 - 1e-12 there)."""
    fft = default_fft(fs)
    out = []
    for j, fp in enumerate((2.5, 10.0)):
        L = 24
        rng = np.random.default_rng([fs, j, 11])
        f0 = rng.uniform(150.0, 230.0, size=L)
        f0[4:10] = 0.0
        f0[14:21] = 0.0
        ap = rng.uniform(0.01, 0.9, size=(L, fft // 2 + 1))
        c = Case("unvoiced pulses", fs, fft, fp, f0, envelope(rng, fs, fft, L), ap, int(L * fp / 1000.0 * fs))
        assert (~c.tb.voiced[c.tb.idx]).sum() > 5
        out.append(c)
    return out


FAMILIES = {"floor": floor_cases, "endpoint": endpoint_cases, "vuv": vuv_cases, "pulses": pulse_cases,
            "nonfinite": nonfinite_cases, "ap_clamp": ap_clamp_cases, "ap_drop": ap_drop_cases,
            "env_sign": env_sign_cases, "env_extreme": env_extreme_cases, "unvoiced": unvoiced_cases}


def check_family(world, ref, family, fs):
    return run_cases(world, ref, family, FAMILIES[family](fs))


# ------------------------------------------------------------------------------------------------------ C. coded rows
def mean_ref(row):
    """CheckVUV's mean (codec.cpp:33-38): the values summed in index order, then divided by their count"""
    tmp = 0.0
    for v in row:
        tmp += float(v)
    with np.errstate(invalid="ignore"):
        return np.float64(tmp) / np.float64(len(row)) if len(row) else np.float64(np.nan)


def rows_around(base, target=-0.5):
    """base (its last value the largest, so that one of its ulps moves the sum by about one of the sum's) with its last
    value moved ulp by ulp until CheckVUV's mean is exactly `target`; then the same row with the
    last value moved on until the mean first leaves `target` on either side: the nearest means the row can reach below
    and above it (one ulp of -0.5 where the division by the count can land there, a few ulps with 5 bands)"""
    row = np.array(base, dtype=np.float64)
    row[-1] = target * len(row) - np.sum(row[:-1])
    for _ in range(4096):
        m = mean_ref(row)
        if m == target:
            break
        row[-1] = np.nextafter(row[-1], np.inf if m < target else -np.inf)
    assert mean_ref(row) == target, f"no row with mean {target!r} near {base}"
    out = [row]
    for way in (-np.inf, np.inf):
        r = row.copy()
        for _ in range(4096):
            r[-1] = np.nextafter(r[-1], way)
            if mean_ref(r) != target:
                break
        assert mean_ref(r) != target, f"the mean of {base} does not leave {target!r}"
        out.append(r)
    return out


def coded_rows(fs, n_ap, L, rng):
    """Coded aperiodicity rows: the mean exactly -0.5 and the nearest reachable means either side (CheckVUV's
    tmp > -0.5, codec.cpp:40; wb_codec.cu:165), among voiced and unvoiced rows from the codec's range."""
    if n_ap == 0:
        return np.zeros((L, 1))
    bases = {1: [[-0.3]], 2: [[-0.25, -0.8], [-0.9, 0.1]], 5: [[1.2, 0.1, -0.8, -0.2, -2.8], [-0.1, -0.7, -0.6, -0.3, -0.8]]}
    special = np.array([r for base in bases[n_ap] for r in rows_around(base)])
    means = [mean_ref(r) for r in special]
    assert -0.5 in means and min(means) < -0.5 < max(means)
    if n_ap <= 2:
        assert down(-0.5) in means and up(-0.5) in means
    c = rng.uniform(-25.0, -1.0, size=(L, n_ap))
    c[::5] = -1e-12                                    # unvoiced frames as CodeAperiodicity writes them
    k = np.arange(L)
    c[k % 3 == 1] = special[(k[k % 3 == 1] // 3) % len(special)]
    return c


def check_coded(world, ref, fs):
    """C11: coded aperiodicity rows whose mean is exactly -0.5 and one ulp either side, at n_ap 0 (8 kHz: the mean is
    0 / 0), 1, 2 and 5 bands.  decode_aperiodicity equals the reference's DecodeAperiodicity; synthesis_coded equals
    decode + synthesis bit for bit, through the lone call, the _options batch and the _packed batch, and is within the
    local bound of the reference's Synthesis on its own decoded rows; the int16 call is pcm16 of the float64 call."""
    n_ap = world.number_of_aperiodicities(fs)
    assert n_ap == ref.number_of_aperiodicities(fs)
    sizes = [default_fft(fs), default_fft(fs) * 2]
    mk = lambda a: pc.make(world, a)
    worst = 0.0
    cases = []
    for j, (fft, fp) in enumerate(zip(sizes, (5.0, 2.5))):
        rng = np.random.default_rng([fs, j, 12])
        L = 36
        dims = min(fft // 4 + 1, 40)
        f0 = rng.uniform(130.0, 250.0, size=L)
        f0[10:13] = 0.0
        sp = envelope(rng, fs, fft, L)
        csp = pc.to_np(world.code_spectral_envelope(mk(sp[None]), fs, fft, dims))[0]
        if j == 1:
            csp[20:23, 0] = -1e5                      # decodes to a zero envelope: the NaN responses of B9
        cap = coded_rows(fs, n_ap, L, rng)
        want_ap = ref.decode_aperiodicity(cap, fs, fft)
        got_ap = pc.to_np(world.decode_aperiodicity(mk(cap[None]), fs, fft))[0]
        world.synchronize()
        # the V/UV decision is exact (the same sum in the same order); the values differ at most by pow's rounding
        err = np.abs(got_ap - want_ap) / np.abs(want_ap)
        assert err.max() <= 1e-12, f"decode_aperiodicity fs {fs} fft {fft}: {err.max():.3e} at frame " \
                                   f"{np.unravel_index(np.argmax(err), err.shape)[0]}"
        dims_sp = ref.decode_spectral_envelope(csp, fs, fft, dims)
        y_len = int(L * fp / 1000.0 * fs)
        cases.append((fft, fp, dims, f0, csp, cap, dims_sp, want_ap, y_len))
    for fft, fp, dims, f0, csp, cap, dsp_r, dap_r, y_len in cases:
        what = f"coded fs {fs} fft {fft} fp {fp}"
        capd = mk(cap[None]) if n_ap > 0 else None
        y = pc.to_np(world.synthesis_coded(mk(f0[None]), mk(csp[None]), capd, fft, fp, fs, y_len))[0]
        y16 = pc.to_np(world.synthesis_coded(mk(f0[None]), mk(csp[None]), capd, fft, fp, fs, y_len, dtype="int16"))[0]
        yo = pc.to_np(world.synthesis_coded(mk(f0[None]), mk(csp[None]), capd, [fft], fp, fs, y_len))[0]
        fo = [0, len(f0)]
        yp = pc.to_np(world.synthesis_coded_packed(mk(f0), mk(csp), mk(cap) if n_ap > 0 else None, fo, fft, fp, fs,
                                                   [0, y_len]))
        dsp = world.decode_spectral_envelope(mk(csp[None]), fs, fft, dims)
        dap = world.decode_aperiodicity(mk(cap[None]), fs, fft)
        yd = pc.to_np(world.synthesis(mk(f0[None]), dsp, dap, fft, fp, fs, y_len))[0]
        world.synchronize()
        assert_same(y, yd, what + ": synthesis_coded vs decode + synthesis")
        assert_same(yo, y, what + ": _options vs lone call")
        assert_same(yp, y, what + ": _packed vs lone call")
        assert np.array_equal(y16, pcm16(y)), what + ": int16 call vs pcm16 of the float64 call"
        nan = np.isnan(y)
        if fft == sizes[1]:
            assert nan.any(), what + ": the zero envelope gave no NaN sample"
            assert (y16[nan] == 0).all()
        yr = ref.synthesis(f0, dsp_r, dap_r, fft, fp, fs, y_len)
        worst = max(worst, local_error(y, yr, fft, what))
    _note("coded worst |y - yr| / local peak", worst)
    return worst
