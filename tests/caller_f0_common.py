"""StoneMask, CheapTrick and D4C on a caller's own F0 and time axis: constructed tables aimed at the kernels' guards and
thresholds, at every rate the stages accept, run through three call forms that must agree bit for bit (the padded
one-option call of each utterance on its own, the padded per-utterance _options call of the whole batch, and the
_packed call with the caller's own frame offsets) and compared frame by frame with the reference.  The same assertions
run against the host emulation (CPU) and the CUDA library (-m gpu).

The tables (each value names the kernel line it is aimed at):
  StoneMask (wb_stonemask.cu)   f0 = 40 and one ulp above, fs/12 and one ulp above (:80); f0 with 1.5 fs/f0 + 1 an
      exact integer and one ulp either side (h and the transform size, :85-89); times whose window indices
      (t + (j - h)/fs) fs fall on exact half samples (round_half_away ties, :96); windows off either end of the signal
      (:110); tones at 0.5 ... 3 times the given f0 (the 2 f0 rejection and the 20 % fallback, :117-118); f0 up to
      fs/12 (harmonic bins clamped at nfft/2, :40); digital silence (pw == 0, :64).
  CheapTrick (wb_cheaptrick.cu) every fft_size the 500 Hz stand-in fits, 2^k up to 8192; f0 at the size's floor
      (replaced by 500 Hz) and one ulp above (:43); negative and zero f0; f0 with 1.5 fs/f0 an exact half integer
      and one ulp either side (the round_half_away tie of h, :116); f0 whose smoothing boundary 2/3 f0 N/fs is an
      exact integer; f0 up to just under 3/8 fs, the widest smoothing the kernel holds (wb_spectral.cuh:86); window
      origins before the signal and past its end (:122, :137).
  D4C (wb_d4c.cu)               negative and zero f0 (the reference skips only f0 == 0, d4c.cpp:274, 386; kernel :226)
      and f0 under 40 / 47 Hz and one ulp either side of 47 (max(40, .) / max(47, .), :237, :264, :465, :619); f0 up to
      just under fs/4, the widest smoothing D4C's kernels hold; thresholds of 0.85, -1 (every voiced frame through the
      general body) and exactly the reference's ap0 of one frame (the ap0 > threshold knife edge, :257).
  Time axes: hops of 1, 2.5, 5.5 and 20 ms; non-monotone and repeated times; utterances of 1, 2, 3 and nwin - 1
      samples.

Above those smoothing widths (and at or above fs/2) the kernels refuse the frame with a status error where the
reference still defines a row: check_refused pins that documented behaviour, with NaN guard cells around the rows."""
import os

import numpy as np
import pytest

import packed_stages_common as ps
import test_parity_common as pc
from refworld import rel_err
from world_b200.api import WorldError

RATES = [8000, 11025, 16000, 22050, 24000, 44100, 48000]
HOPS = [1.0, 2.5, 5.5, 20.0]
TOL = 1e-6
CODED_TOL = 1e-9            # coded rows against code_* of the full rows (coded_batch_common.py)
EPS = np.finfo(np.float64).eps

# worst values seen, per stage and rate (printed by report(); pytest -s shows them)
STATS = {}


def _note(key, value):
    STATS[key] = max(STATS.get(key, 0.0), float(value))


def report():
    for k in sorted(STATS):
        print(f"caller f0: {k}: {STATS[k]:.3g}")


def up(v):
    return float(np.nextafter(v, np.inf))


def down(v):
    return float(np.nextafter(v, -np.inf))


def voice(fs, n, f_base=180.0, seed=0, tone=None):
    """A harmonic voice (or one pure tone at `tone` Hz) with a little noise, n samples."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    if tone is not None:
        return np.sin(2 * np.pi * tone * t) * 0.5 + rng.standard_normal(n) * 1e-4
    x = np.zeros(n)
    for k in range(1, 30):
        if k * f_base < fs / 2:
            x += np.sin(2 * np.pi * k * f_base * t + 0.3 * k) / k
    return x * 0.3 + rng.standard_normal(n) * 1e-3


def hop_times(n, fs, hop_ms):
    k = int(1000.0 * n / fs / hop_ms) + 1
    return np.arange(k) * hop_ms / 1000.0


def special_times(n, fs):
    """Before the signal, past its end, repeated, non-monotone, and a CheapTrick origin tie (t fs + 0.001 = m + 0.5)."""
    d = n / fs
    return np.array([0.0, -0.004, -1.0, d, d + 0.003, d + 1.0, 0.5 * d, 0.5 * d, 0.25 * d, 0.75 * d, 0.1 * d,
                     (int(0.3 * n) + 0.5 - 0.001) / fs])


def table(hop, special, f0s):
    """Frames pairing every value of f0s with a time on the hop grid (the grid repeated as needed: repeated times) and
    again with the special times."""
    grid = np.resize(hop, max(len(hop), len(f0s)))
    t = np.concatenate([grid, special])
    f0 = np.concatenate([np.resize(np.array(f0s, dtype=np.float64), len(grid)),
                         np.resize(np.array(f0s, dtype=np.float64)[::-1], len(special))])
    return t, f0


class Utts:
    """Utterances (x, t, f0) back to back, with what each call form needs."""

    def __init__(self, world, fs, utts):
        self.world, self.fs, self.utts = world, fs, utts
        self.lens = [len(u[0]) for u in utts]
        self.frames = [len(u[1]) for u in utts]
        self.xo = np.concatenate([[0], np.cumsum(self.lens)]).astype(np.int64)
        self.fo = np.concatenate([[0], np.cumsum(self.frames)]).astype(np.int64)
        mk = lambda a: pc.make(world, a)
        self.x = mk(np.concatenate([u[0] for u in utts]))
        self.t_np = np.concatenate([u[1] for u in utts]).astype(np.float64)
        self.f0_np = np.concatenate([u[2] for u in utts]).astype(np.float64)
        self.t, self.f0 = mk(self.t_np), mk(self.f0_np)
        L, n = max(self.lens), len(utts)
        xr = np.zeros((n, L))
        for u, (x, _, _) in enumerate(utts):
            xr[u, :len(x)] = x
        self.x_rows = mk(xr)
        self.t_rows = mk(ps.padded(self.t_np, self.fo))
        self.f0_rows = mk(ps.padded(self.f0_np, self.fo))
        self.kw = dict(x_lengths=self.lens, f0_lengths=self.frames)

    def lone(self, u):
        """utterance u as a batch of one: the arguments x, fs, time_axis, f0"""
        x, t, f0 = self.utts[u]
        mk = lambda a: pc.make(self.world, np.asarray(a, dtype=np.float64)[None])
        return mk(x), self.fs, mk(t), mk(f0)

    def rows(self, a, u, width=None):
        a = pc.to_np(a)
        r = a[self.fo[u]:self.fo[u + 1]]
        return r if width is None else r[:, :width]


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, f"{what}: shapes {a.shape} {b.shape}"
    bad = np.argwhere(a.view(np.uint64) != b.view(np.uint64))
    assert bad.size == 0, f"{what}: differs at {bad[:4].tolist()}"


# ------------------------------------------------------------------------------------------------------------ CheapTrick
def ct_sizes(fs):
    """Every fft_size CheapTrick defines at fs: the 500 Hz stand-in's window 2 round(1.5 fs / 500) + 1 fits, up to
    the library's 8192."""
    need = 2 * int(1.5 * fs / 500.0 + 0.5) + 1
    return [1 << k for k in range(4, 14) if (1 << k) >= need]


def ct_f0s(fs, N):
    """CheapTrick's F0 table at one size (module docstring)."""
    floor = 3.0 * fs / (N - 3.0)
    top = 0.375 * fs * (1 - 4.0 / N)                  # below the widest smoothing the kernel holds
    v = [floor, up(floor), -50.0, 0.0, 500.0, 0.37 * fs if N >= 64 else 0.3 * fs, top * (1 - 1e-9)]
    kmax = int(1.5 * fs / floor)
    for k in sorted({kmax - 1, max(5, kmax // 2), max(5, kmax // 5), 6}):
        f = 1.5 * fs / (k + 0.5)                       # 1.5 fs / f = k + 0.5: h's rounding tie
        if floor < f < top:
            v += [f, down(f), up(f)]
    for m in (N // 8, N // 5, N // 16):
        f = 1.5 * m * fs / N                           # smoothing boundary 2/3 f N / fs = m
        if floor < f < top:
            v += [f, up(f)]
    return [x for x in v if x < top]


def ct_utts(fs):
    """One utterance per fft_size, each at its own hop, plus utterances of 1, 2, 3 and nwin - 1 samples."""
    out = []
    for s, N in enumerate(ct_sizes(fs)):
        n = int(0.06 * fs)
        x = voice(fs, n, f_base=120.0 + 40 * s, seed=s)
        f0s = ct_f0s(fs, N)
        t, f0 = table(hop_times(n, fs, HOPS[s % len(HOPS)])[:24], special_times(n, fs), f0s)
        out.append((N, (x, t, f0)))
    N = ct_sizes(fs)[0]
    floor = 3.0 * fs / (N - 3.0)
    nwin = 2 * int(1.5 * fs / 500.0 + 0.5) + 1
    for n in (1, 2, 3, nwin - 1):
        x = voice(fs, n, seed=n)
        t = np.array([0.0, n / fs / 2, -0.001, 1.0])
        out.append((N, (x, t, np.array([200.0 + floor, 0.0, up(floor), 0.3 * fs]))))
    return out


def check_cheaptrick(world, ref, fs):
    """The three call forms bit for bit, the coded forms against code_spectral_envelope of the full rows, and every
    frame within 1e-6 of the reference."""
    cases = ct_utts(fs)
    sizes = [N for N, _ in cases]
    U = Utts(world, fs, [u for _, u in cases])
    opts = []
    for N in sizes:
        o = world.cheaptrick_option(fs)
        o.fft_size = N
        opts.append(o)
    W = max(sizes) // 2 + 1
    packed = world.cheaptrick_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, opts)
    batch = world.cheaptrick(U.x_rows, fs, U.t_rows, U.f0_rows, opts, **U.kw)
    dims = min(ps.DIMS, min(sizes) // 4 + 1)
    coded = world.cheaptrick_coded_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, dims, opts)
    world.synchronize()
    worst = 0.0
    for u, N in enumerate(sizes):
        b = N // 2 + 1
        x, t, f0 = U.utts[u]
        lone = pc.to_np(world.cheaptrick(*U.lone(u), opts[u]))[0]
        world.synchronize()
        got = U.rows(packed, u, b)
        assert_same(got, lone, f"cheaptrick fs {fs} N {N}: packed vs lone call")
        assert_same(pc.to_np(batch)[u, :len(t), :b], lone, f"cheaptrick fs {fs} N {N}: _options vs lone call")
        assert np.isnan(got).sum() == 0
        o = ref.cheaptrick_option(fs)
        o.fft_size = N
        want = ref.cheaptrick(x, fs, t, f0, o)
        r = rel_err(got, want).max()
        worst = max(worst, r)
        assert r < TOL, f"cheaptrick fs {fs} N {N} vs reference: {r:.3e} at frame {np.argmax(rel_err(got, want).max(1))}"
        want_c = pc.to_np(world.code_spectral_envelope(pc.make(world, got[None]), fs, N, dims))[0]
        pc.assert_close_signed(U.rows(coded, u), want_c, f"cheaptrick coded fs {fs} N {N}", tol=CODED_TOL)
    _note(f"cheaptrick max rel err vs reference, {fs} Hz", worst)


# ------------------------------------------------------------------------------------------------------------------ D4C
D4C_REF_MIN_FS = 12000      # below, the reference corrupts its own heap (tests/test_d4c_body_sizes.py)


def d4c_fft(fs):
    return int(2 ** (1 + int(np.log(4.0 * fs / 47.0 + 1) / np.log(2))))


def d4c_f0s(fs):
    top = 0.25 * fs * (1 - 4.0 / d4c_fft(fs))          # below the widest smoothing D4C's kernels hold
    return [-300.0, -1e-3, 0.0, 30.0, 39.9, 40.0, up(40.0), 46.9, down(47.0), 47.0, up(47.0), 120.0, 245.0, 700.0,
            0.1 * fs, top * (1 - 1e-9), -0.0]


def ref_ap0(ref, x, fs, t, f0, N, k):
    """The reference's LoveTrain ap0 of frame k, to the last bit: the smallest threshold at which frame k is not
    selected (ap0 is computed for every frame before any general body runs, so it does not depend on the threshold)."""
    unsel = 1.0 - 1e-12                              # InitializeAperiodicity's fill (kMySafeGuardMinimum)

    def selected(th):
        d = ref.d4c_option()
        d.threshold = th
        return ref.d4c(x, fs, t, f0, N, d)[k, 0] != unsel

    lo, hi = np.float64(0.0).view(np.int64), np.float64(1.0).view(np.int64)
    assert selected(0.0) and not selected(1.0)
    while hi - lo > 1:                               # selected(lo), not selected(hi)
        mid = (lo + hi) // 2
        if selected(np.int64(mid).view(np.float64)):
            lo = mid
        else:
            hi = mid
    return float(np.int64(hi).view(np.float64))


def d4c_utts(fs, ref):
    """Utterances with thresholds 0.85 (default), -1 and the knife edge; sizes alternate between two CheapTrick
    sizes.  Returns [(fft_size, threshold, (x, t, f0))], and the knife-edge utterance's index."""
    sizes = ct_sizes(fs)
    pick = [sizes[0], sizes[min(2, len(sizes) - 1)]]
    out = []
    f0s = d4c_f0s(fs)
    for s, (th, hop) in enumerate(((0.85, 5.5), (-1.0, 2.5), (-1.0, 20.0), (0.85, 1.0))):
        n = int(0.05 * fs)
        x = voice(fs, n, f_base=110.0 + 60 * s, seed=10 + s)
        t, f0 = table(hop_times(n, fs, hop)[:16], special_times(n, fs), f0s)
        out.append((pick[s % 2], th, (x, t, f0)))
    for n in (1, 2, 3):
        out.append((pick[0], -1.0, (voice(fs, n, seed=n), np.array([0.0, 0.01]), np.array([150.0, -20.0]))))
    # the knife edge: threshold exactly the reference's ap0 of frame 2 (not selected there: ap0 > ap0 fails)
    n = int(0.03 * fs)
    x = voice(fs, n, f_base=210.0, seed=20)
    x = x + np.random.default_rng(22).standard_normal(n) * 0.05
    t = hop_times(n, fs, 5.0)
    f0 = np.full(len(t), 210.0)
    knife = None
    if ref is not None and fs >= D4C_REF_MIN_FS:
        knife = ref_ap0(ref, x, fs, t, f0, pick[0], 2)
    out.append((pick[0], knife if knife is not None else 0.5, (x, t, f0)))
    return out, len(out) - 1


def check_d4c(world, ref, fs):
    """The three call forms bit for bit, the coded forms against code_aperiodicity of the full rows, and (from 12 kHz)
    every frame within 1e-6 of the reference.  At the knife edge the library may take either side of ap0 > threshold
    (its ap0 is a different rounding of the same sum); its rows must then equal the reference's on that side."""
    with_ref = ref is not None and fs >= D4C_REF_MIN_FS
    cases, ki = d4c_utts(fs, ref if with_ref else None)
    sizes = [N for N, _, _ in cases]
    U = Utts(world, fs, [u for _, _, u in cases])
    opts = []
    for _, th, _ in cases:
        d = world.d4c_option()
        d.threshold = th
        opts.append(d)
    packed = world.d4c_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, sizes, opts)
    batch = world.d4c(U.x_rows, fs, U.t_rows, U.f0_rows, sizes, opts, **U.kw)
    n_ap = world.number_of_aperiodicities(fs)
    coded = world.d4c_coded_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, sizes, opts) if n_ap > 0 else None
    world.synchronize()
    worst, knife_flips = 0.0, 0
    for u, (N, th, (x, t, f0)) in enumerate(cases):
        b = N // 2 + 1
        lone = pc.to_np(world.d4c(*U.lone(u), N, opts[u]))[0]
        world.synchronize()
        got = U.rows(packed, u, b)
        assert_same(got, lone, f"d4c fs {fs} utterance {u}: packed vs lone call")
        assert_same(pc.to_np(batch)[u, :len(t), :b], lone, f"d4c fs {fs} utterance {u}: _options vs lone call")
        assert np.isfinite(got).all()
        if n_ap > 0:
            want_c = pc.to_np(world.code_aperiodicity(pc.make(world, got[None]), fs, N))[0]
            pc.assert_close_signed(U.rows(coded, u), want_c[:, :n_ap], f"d4c coded fs {fs} utterance {u}",
                                   tol=CODED_TOL)
        if not with_ref:
            continue
        d = ref.d4c_option()
        d.threshold = th
        want = ref.d4c(x, fs, t, f0, N, d)
        r = rel_err(got, want).max()
        if u == ki:
            assert want[2, 0] == 1.0 - 1e-12, "the knife edge: the reference does not select frame 2"
            d.threshold = down(th)
            other = ref.d4c(x, fs, t, f0, N, d)
            assert other[2, 0] != want[2, 0], "the knife edge: one ulp lower the reference selects frame 2"
            r2 = rel_err(got, other).max()
            if r2 < r:
                knife_flips += 1
                r = r2
            # a threshold a hair off the edge leaves no choice
            for thx, ref_th in ((th * (1 + 1e-9), th), (th * (1 - 1e-9), down(th))):
                dd = world.d4c_option()
                dd.threshold = thx
                g = pc.to_np(world.d4c(*U.lone(u), N, dd))[0]
                d.threshold = ref_th
                assert rel_err(g, ref.d4c(x, fs, t, f0, N, d)).max() < TOL, f"d4c fs {fs}: threshold {thx!r}"
        worst = max(worst, r)
        assert r < TOL, f"d4c fs {fs} utterance {u} vs reference: {r:.3e} at frame {np.argmax(rel_err(got, want).max(1))}"
    world.synchronize()
    if with_ref:
        _note(f"d4c max rel err vs reference, {fs} Hz", worst)
        _note("d4c knife-edge frames decided the other way", knife_flips)


# ------------------------------------------------------------------------------------------------------------ StoneMask
def sm_window_size(fs, f0):
    h = int(1.5 * fs / f0 + 1.0)
    nwin = 2 * h + 1
    return h, nwin, 1 << (2 + int(np.floor(np.log2(nwin))))


def matlab_round(v):
    v = np.asarray(v, dtype=np.float64)
    return np.where(v > 0, np.trunc(v + 0.5), np.trunc(v - 0.5)).astype(np.int64)


def sm_restate(x, fs, t, f0):
    """GetRefinedF0 (stonemask.cpp:187-208) in np.longdouble for one frame: the window indices rounded as the
    reference rounds them (in double), Blackman and differentiated windows, the <= 8 DFT bins FixF0 reads as explicit
    sums, FixF0 twice and both decisions.  Returns (refined f0, bound, knife) where `knife` is True if a decision or a
    harmonic bin's rounding lies within the bound of its threshold (either outcome is then accepted).

    The bound: each bin X = sum_j s_j w_j e^{-i theta_j} is computed by the library (sparse DFT) and the reference
    (FFT) with an error of at most c n eps sum_j |s_j w_j| (n = 2h + 1 terms, c = 8 covering the window values' own
    rounding); a harmonic's instantaneous frequency k fs/N + Im(conj(M) D)/|M|^2 fs/(2 pi) then moves by at most
    fs/(2 pi) (dD/|M| + 2 |D| dM/|M|^2), its amplitude |M| by dM, and FixF0's ratio of sums accordingly (first
    order, summed over the six harmonics), plus 16 eps of the result for the final arithmetic."""
    L = np.longdouble
    if f0 <= 40.0 or f0 > fs / 12.0:
        return 0.0, 0.0, False
    h, nwin, nfft = sm_window_size(fs, f0)
    j = np.arange(nwin)
    r = matlab_round((t + (j - h).astype(np.float64) / fs) * fs)
    T = L(2 * h + 1) / L(fs)
    tmp = (r.astype(L) - L(1)) / L(fs) - L(t)
    pi = L(np.pi) + L(1.2246467991473532e-16)
    w = L(0.42) + L(0.5) * np.cos(2 * pi * tmp / T) + L(0.08) * np.cos(4 * pi * tmp / T)
    dw = np.empty(nwin, dtype=L)
    dw[0] = -w[1] / 2
    dw[1:-1] = -(w[2:] - w[:-2]) / 2
    dw[-1] = w[-2] / 2
    s = np.asarray(x, dtype=np.float64)[np.clip(r - 1, 0, len(x) - 1)].astype(L)
    if not s.any():
        # digital silence: every bin is exactly 0 in any evaluation (pw == 0), FixF0 gives 0, the tentative F0 is
        # rejected and the frame keeps f0 -- exact, no bound
        return float(f0), 0.0, False
    xw, xd = s * w, s * dw
    err_m = 8 * nwin * EPS * float(np.abs(xw).sum())
    err_d = 8 * nwin * EPS * float(np.abs(xd).sum())

    def bin_of(f, m):
        return min(int(matlab_round(f * nfft / fs * (m + 1))), nfft // 2)

    def tie_margin(f, m, df):
        """True if bin m's rounding could go either way for f within df"""
        v = f * nfft / fs * (m + 1)
        return abs(v - np.floor(v) - 0.5) <= df * nfft / fs * (m + 1) + 4 * EPS * abs(v)

    def fix(f_init, H, df_init):
        num, den, bnum, bden, knife = L(0), L(0), 0.0, 0.0, False
        for m in range(H):
            k = bin_of(f_init, m)
            knife |= tie_margin(f_init, m, df_init)
            ang = 2 * pi * L(1) * ((k * j) % nfft).astype(L) / L(nfft)
            c, sn = np.cos(ang), -np.sin(ang)
            mr, mi = (xw * c).sum(), (xw * sn).sum()
            dr, di = (xd * c).sum(), (xd * sn).sum()
            pw = mr * mr + mi * mi
            amp = np.sqrt(pw)
            inst = L(0) if pw == 0 else L(k) * fs / nfft + (mr * di - mi * dr) / pw * fs / 2 / pi
            num += amp * inst
            den += amp * (m + 1)
            a, dmag = float(amp), float(np.sqrt(dr * dr + di * di))
            d_inst = np.inf if a <= err_m else fs / (2 * np.pi) * (err_d / a + 2 * dmag * err_m / a ** 2)
            bnum += a * d_inst + abs(float(inst)) * err_m
            bden += (m + 1) * err_m
        res = num / (den + L(1e-12))      # kMySafeGuardMinimum
        den_f = float(den)
        bound = np.inf if den_f <= bden else (bnum + abs(float(res)) * bden) / (den_f - bden) + 16 * EPS * abs(float(res))
        return float(res), bound, knife

    tent, b1, knife = fix(f0, 2, 0.0)
    if tent <= 0.0 or tent > f0 * 2:
        if abs(tent) <= b1 or abs(tent - 2 * f0) <= b1:
            knife = True
        mean, b2 = 0.0, 0.0
    else:
        if abs(tent) <= b1 or abs(tent - 2 * f0) <= b1:
            knife = True
        mean, b2, k2 = fix(tent, 6, b1)
        knife |= k2
    if abs(abs(mean - f0) - f0 * 0.2) <= b2 + 4 * EPS * f0:
        knife = True
    if abs(mean - f0) > f0 * 0.2:
        return float(f0), 0.0, knife
    return mean, b2, knife


def sm_utts(fs):
    """StoneMask's table (module docstring): a voice, tones at ratios of the given f0, and digital silence."""
    n = int(0.08 * fs)
    out = []
    top = fs / 12.0
    v = [40.0, up(40.0), 39.0, top, up(top), down(top), 0.9 * top, -100.0, 0.0, 180.0, 360.0, 90.0, 45.0]
    for k in (4, 7, 20, 60, int(1.5 * fs / 41.0) + 1):
        f = 1.5 * fs / (k - 1)                         # 1.5 fs / f + 1 = k
        if 40.0 < f <= top:
            v += [f, down(f), up(f)]
    x = voice(fs, n, f_base=180.0, seed=1)
    t = np.concatenate([hop_times(n, fs, HOPS[0])[::4], special_times(n, fs)])
    # half-sample ties of the window indices: t = (m + 0.5) / fs for which some (t + (j - h)/fs) fs lands on .5
    ties = []
    for m in range(int(0.2 * n), int(0.8 * n)):
        tt = (m + 0.5) / fs
        h, nwin, _ = sm_window_size(fs, 180.0)
        q = (tt + (np.arange(nwin) - h).astype(np.float64) / fs) * fs
        if np.any(q - np.floor(q) == 0.5):
            ties.append(tt)
        if len(ties) == 6:
            break
    t = np.concatenate([t, ties, ties])
    f0 = np.resize(np.array(v), len(t))
    f0[-2 * len(ties):] = np.resize([180.0, 179.0, 181.0], 2 * len(ties))
    out.append((x, t, f0))
    # tones at ratios of the given f0: the 2 f0 rejection and the 20 % fallback on either side
    ratios = [0.5, 0.78, 0.8, 0.82, 1.0, 1.18, 1.2, 1.22, 1.5, 1.95, 2.0, 2.05, 3.0]
    for s, base in enumerate((150.0, min(600.0, 0.8 * top))):
        xs = voice(fs, n, seed=2 + s, tone=base)
        ts = np.resize(hop_times(n, fs, 5.5)[2:-2], len(ratios))
        out.append((xs, ts, base / np.array(ratios)))
    out.append((np.zeros(n), hop_times(n, fs, 20.0), np.full(len(hop_times(n, fs, 20.0)), 200.0)))
    for m in (1, 2, 3, sm_window_size(fs, 200.0)[1] - 1):
        out.append((voice(fs, m, seed=m), np.array([0.0, m / fs, -0.01]), np.array([200.0, 41.0, up(top) / 1.5])))
    return out


def check_stonemask(world, ref, fs):
    """The padded call and the packed call bit for bit; every frame within its bound (sm_restate) of the long-double
    restatement, on the restatement's branch wherever the decisions' margins exceed the bound; the restatement within
    the same bound of the reference."""
    U = Utts(world, fs, sm_utts(fs))
    packed = world.stonemask_packed(U.x, U.xo, fs, U.t, U.f0, U.fo)
    batch = world.stonemask(U.x_rows, fs, U.t_rows, U.f0_rows, **U.kw)
    world.synchronize()
    worst_frac, knives = 0.0, 0
    for u, (x, t, f0) in enumerate(U.utts):
        got = U.rows(packed, u)
        assert_same(pc.to_np(batch)[u, :len(t)], got, f"stonemask fs {fs} utterance {u}: padded vs packed")
        lone = pc.to_np(world.stonemask(*U.lone(u)))[0]
        assert_same(lone, got, f"stonemask fs {fs} utterance {u}: lone vs packed")
        want_ref = ref.stonemask(x, fs, t, f0) if ref is not None else None
        for i in range(len(t)):
            exact, bound, knife = sm_restate(x, fs, float(t[i]), float(f0[i]))
            if want_ref is not None:
                assert abs(want_ref[i] - exact) <= bound or knife, \
                    f"restatement vs reference fs {fs} utt {u} frame {i}: {want_ref[i]!r} {exact!r} bound {bound:.3g}"
            if knife:
                knives += 1
                continue
            err = abs(got[i] - exact)
            assert err <= bound, f"stonemask fs {fs} utt {u} frame {i} (f0 {f0[i]!r}, t {t[i]!r}): {got[i]!r} vs " \
                                 f"{exact!r}, bound {bound:.3g}"
            if bound > 0:
                worst_frac = max(worst_frac, err / bound)
    _note(f"stonemask worst error / bound, {fs} Hz", worst_frac)
    _note(f"stonemask knife-edge frames, {fs} Hz", knives)


# ------------------------------------------------------------------------------------------------ where it is undefined
def check_refused(world, fs):
    """Frames the kernels refuse (f0 at or above fs/2, and the smoothing widths they cannot hold, where the reference
    still defines a row; CheapTrick's window longer than fft_size) fail the call with a status error; the other
    frames' rows are written, and nothing is written past frames [0, F) or past fft_size / 2 + 1 (NaN guard cells).

    The refused values include f0 = (0.5 - 1.5/N) fs, inside the window between two and one bin below Nyquist where
    dc_correction's clamp differs from the reference (wb_spectral.cuh), at two CheapTrick sizes and at D4C's own
    transform size: the frame is refused, so no row shaped by the clamp is kept.

    The status error does not name the utterance: the device status word collects every call queued on the context
    since the last synchronize and is read only there, so an utterance index recorded by the kernel could not say which
    of those calls it belongs to."""
    n = int(0.04 * fs)
    x = voice(fs, n, seed=40)
    good_t, good_f = np.array([0.01, 0.02]), np.array([150.0, 300.0])
    for N in (ct_sizes(fs)[-2], ct_sizes(fs)[0]):
        o = world.cheaptrick_option(fs)
        o.fft_size = N
        check_refused_cheaptrick(world, fs, x, N, o, good_t, good_f, with_d4c=N == ct_sizes(fs)[-2])
    # D4C between fs/4 and fs/2, and inside the dc_correction window of its own transform size
    if fs >= D4C_REF_MIN_FS:
        Nd = d4c_fft(fs)
        for bad in (0.26 * fs, (0.5 - 1.5 / Nd) * fs):
            U = Utts(world, fs, [(x, np.array([0.01]), np.array([bad]))])
            d = world.d4c_option()
            d.threshold = -1.0
            world.d4c_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, [ct_sizes(fs)[-2]], [d])
            with pytest.raises(WorldError, match="smoothing width"):
                world.synchronize()
    # CheapTrick's window longer than fft_size: a size too small for the 500 Hz stand-in
    small = ct_sizes(fs)[0] // 2
    if small >= 16:
        o2 = world.cheaptrick_option(fs)
        o2.fft_size = small
        U = Utts(world, fs, [(x, np.array([0.01]), np.array([0.0]))])
        world.cheaptrick_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, [o2])
        with pytest.raises(WorldError, match="window longer than fft_size"):
            world.synchronize()
    # the context works afterwards
    o = world.cheaptrick_option(fs)
    want = pc.to_np(world.cheaptrick(pc.make(world, x[None]), fs, pc.make(world, good_t[None]),
                                     pc.make(world, good_f[None]), o))
    world.synchronize()
    assert np.isfinite(want).all()


def check_refused_cheaptrick(world, fs, x, N, o, good_t, good_f, with_d4c):
    """check_refused at one CheapTrick size (with_d4c: the same frames through D4C)"""
    for bad, pattern in ((0.5 * fs, "smoothing width"), (0.49 * fs, "smoothing width"), (2.0 * fs, "smoothing width"),
                         (np.inf, "smoothing width"), (0.376 * fs, "smoothing width"),
                         ((0.5 - 1.5 / N) * fs, "smoothing width")):
        t = np.array([0.01, 0.015, 0.02])
        f0 = np.array([150.0, bad, 300.0])
        U = Utts(world, fs, [(x, t, f0)])
        W, F = N // 2 + 1 + 3, 3
        out = pc.make(world, np.full((F + 2, W), np.nan))
        world.cheaptrick_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, [o], out=out)
        with pytest.raises(WorldError, match=pattern):
            world.synchronize()
        g = pc.to_np(out)
        assert np.isnan(g[F:]).all() and np.isnan(g[:, N // 2 + 1:]).all(), f"cheaptrick f0 {bad}: guard cells"
        assert np.isnan(g[1]).all(), f"cheaptrick f0 {bad}: the refused frame's row"
        want = pc.to_np(world.cheaptrick(pc.make(world, x[None]), fs, pc.make(world, good_t[None]),
                                         pc.make(world, good_f[None]), o))[0]
        world.synchronize()
        # the frame before the refused one is the call's without it (later frames' noise draws come after the refused
        # frame's, as in the reference)
        assert_same(g[0, :N // 2 + 1], want[0], f"cheaptrick f0 {bad}: the frame before")
        assert np.isfinite(g[2, :N // 2 + 1]).all(), f"cheaptrick f0 {bad}: the frame after"
        if with_d4c and fs >= D4C_REF_MIN_FS:
            d = world.d4c_option()
            d.threshold = -1.0                             # every voiced frame through the general body
            a = world.d4c_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, [N], [d])
            if np.isinf(bad):               # LoveTrain's ap0 is NaN: the frame is not selected, its row the fill
                world.synchronize()
                assert np.isfinite(pc.to_np(a)).all(), "d4c f0 inf"
                continue
            with pytest.raises(WorldError, match=pattern):
                world.synchronize()


def check_poison(world, fs):
    """Every stage's rows on the constructed tables are bit for bit the same with every scratch block poisoned
    (WB_ARENA_POISON=0xFF: a stale double read is a NaN)."""
    def run():
        U = Utts(world, fs, [u for _, u in ct_utts(fs)][:2])
        opts = []
        for N in ct_sizes(fs)[:2]:
            o = world.cheaptrick_option(fs)
            o.fft_size = N
            opts.append(o)
        sp = pc.to_np(world.cheaptrick_packed(U.x, U.xo, fs, U.t, U.f0, U.fo, opts)).copy()
        cases = d4c_utts(fs, None)[0][:2]
        D = Utts(world, fs, [u for _, _, u in cases])
        opts = []
        for _, th, _ in cases:
            d = world.d4c_option()
            d.threshold = th
            opts.append(d)
        ap = pc.to_np(world.d4c_packed(D.x, D.xo, fs, D.t, D.f0, D.fo, [N for N, _, _ in cases], opts)).copy()
        V = Utts(world, fs, sm_utts(fs)[:2])
        sm = pc.to_np(world.stonemask_packed(V.x, V.xo, fs, V.t, V.f0, V.fo)).copy()
        world.synchronize()
        return sp, ap, sm

    clean = run()
    saved = os.environ.get("WB_ARENA_POISON")
    try:
        os.environ["WB_ARENA_POISON"] = "0xFF"
        got = run()
    finally:
        if saved is None:
            os.environ.pop("WB_ARENA_POISON", None)
        else:
            os.environ["WB_ARENA_POISON"] = saved
    for name, a, b in zip(("cheaptrick", "d4c", "stonemask"), clean, got):
        assert_same(b, a, f"{name} under WB_ARENA_POISON=0xFF, fs {fs}")
