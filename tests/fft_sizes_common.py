"""CheapTrick, D4C, the codec and Synthesis at every FFT size they accept, against the reference.  Each check is written
once and runs on the host emulation (a reduced grid, CPU suite) and on the CUDA library (the full grid, -m gpu).

The default option gives one fft_size per rate (512 at 8 kHz ... 4096 at 96 kHz), but callers reach every other size
through CheapTrickOption.f0_floor or by setting fft_size directly.  The small sizes leave most of a frame kernel's
threads idle, the large ones take the longest shared-memory requests, and in between the codec's DCT shrinks to a few
points; each check therefore sweeps the sizes at several rates on ragged batches (row offsets at every row width).

Where the reference itself is undefined the checks compare the library only with itself:
  * CheapTrick analyses a frame at or below its floor 3 fs / (fft_size - 3) with the 500 Hz window of
    2 round(1.5 fs / 500) + 1 samples, which overruns fft_size below 64 at 8 kHz ... 512 at 48 kHz; the library
    reports WORLD_B200_EDOMAIN there (status bit 1) and must still match when every frame is above the floor.
  * Synthesis writes a pulse interval of noise into an fft_size buffer (synthesis.cpp:19-30), so it is compared with
    the reference only where every interval is at most 0.8 fft_size: voiced f0 >= 1.25 (fs // fft_size + 1) (twice
    that next to unvoiced frames, where the time base halves it) and the 500 Hz pulses of unvoiced frames,
    fs / 500 <= 0.8 fft_size.  A model of the reference's time base checks the intervals before each call.

Tolerances are the project's: 1e-6 relative for envelopes and aperiodicities, assert_close_signed for coded rows,
1e-9 of the waveform peak for Synthesis, bit for bit where two paths of the library must agree, and padded frames and
samples are never written.  Every check returns its worst error per (rate, size)."""
import ctypes as C

import numpy as np
import pytest

from refworld import rel_err
from synthesis_host_common import quantise
from test_parity_common import assert_close, assert_close_signed, make, to_np
from world_b200.api import CheapTrickOption, D4COption, F0_DIO_STONEMASK, F0_HARVEST, WorldError

POW2 = [1 << k for k in range(4, 14)]                    # 16 ... 8192: CheapTrick and the spectral envelope codec
SYNTHESIS_SIZES = POW2[:-1]                              # 16 ... 4096
D4C_SIZES = [4, 16, 64, 256, 1000, 1024, 3001, 4096, 8192]
CT_RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000]
D4C_RATES = [16000, 22050, 24000, 32000, 44100, 48000]   # D4C is undefined in the reference below 15.8 kHz
SYNTHESIS_RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000]
FP = 5.0


def table(worst, what):
    """One line per rate: the worst error at each size."""
    lines = [f"{what}, worst error per (rate, size):"]
    for fs in sorted({k[0] for k in worst}):
        lines.append(f"  {fs:6d} Hz: " + "  ".join(f"{s}: {e:.1e}" for (r, s), e in sorted(worst.items()) if r == fs))
    return "\n".join(lines)


def _batch(fs, seed):
    """Three utterances of 0.5, ~0.37 and ~0.21 s (different lengths at every rate) and their frame counts."""
    from synth import synth_batch
    lens = [fs // 2, int(0.37 * fs) + 13, int(0.21 * fs) + 7]
    x = synth_batch([seed, seed + 1, seed + 2], fs, lens[0]).numpy()
    return x, lens, [int(1000.0 * v / fs / FP) + 1 for v in lens]


def _rows(values, frames):
    """[n, max frames] rows from per-utterance vectors (zero beyond each utterance)."""
    out = np.zeros((len(frames), max(frames)))
    for u, v in enumerate(values):
        out[u, :frames[u]] = v
    return out


def _time_rows(frames):
    return _rows([np.arange(m) * FP / 1000.0 for m in frames], frames)


def _unwritten(a, frames, what):
    for u, m in enumerate(frames):
        assert not a[u, m:].any(), f"{what}: utterance {u}, padded frames were written"


# ---------------------------------------------------------------- 1. sizing helpers
def check_sizing_helpers(world, ref):
    """GetFFTSizeForCheapTrick and GetF0FloorForCheapTrick equal the reference bit for bit, over rates 8 ... 96 kHz and
    f0_floor values that include those where 3 fs / f0_floor + 1 is a power of two, and one ulp either side."""
    lib, rlib = world.lib, ref.lib
    rlib.GetFFTSizeForCheapTrick.argtypes = [C.c_int, C.POINTER(CheapTrickOption)]
    n = 0
    for fs in (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000):
        floors = list(np.geomspace(5.0, 2000.0, 97))
        for p in range(3, 17):
            exact = 3.0 * fs / ((1 << p) - 1)
            floors += [exact, np.nextafter(exact, 0.0), np.nextafter(exact, np.inf)]
        assert any(3.0 * fs / f + 1 == float(1 << p) for f in floors for p in range(3, 17))
        for f in floors:
            o = CheapTrickOption(); o.q1 = -0.15; o.f0_floor = float(f); o.fft_size = 0
            got, want = lib.GetFFTSizeForCheapTrick(fs, C.byref(o)), rlib.GetFFTSizeForCheapTrick(fs, C.byref(o))
            assert got == want, f"GetFFTSizeForCheapTrick({fs}, f0_floor {f!r}): {got}, reference {want}"
            n += 1
        for fft in list(POW2) + [4, 5, 1000, 3001]:
            got, want = lib.GetF0FloorForCheapTrick(fs, fft), rlib.GetF0FloorForCheapTrick(fs, fft)
            assert got == want, f"GetF0FloorForCheapTrick({fs}, {fft}): {got!r}, reference {want!r}"
    return n


# ---------------------------------------------------------------- 2. CheapTrick, plain and fused coded
def ct_floor(fs, fft):
    return 3.0 * fs / (fft - 3.0)                        # GetF0FloorForCheapTrick


def ct_defined(fs, fft):
    """True when the 500 Hz window that frames at or below the floor get fits in fft_size."""
    return 2 * int(np.floor(1.5 * fs / 500.0 + 0.5)) + 1 <= fft


def ct_option(fs, fft, q1=-0.15):
    o = CheapTrickOption()
    o.q1 = q1; o.f0_floor = ct_floor(fs, fft); o.fft_size = fft
    return o


def ct_contours(rng, fs, fft, frames, at_floor):
    """f0 rows: random between floor (1 + 1e-4) (the longest window that fits) and min(1000, fs / 4) -- at least
    1.05 floor where the floor is higher -- with every fifth frame at floor (1 + 1e-4).  at_floor adds unvoiced frames
    and frames exactly at the floor, which CheapTrick analyses at 500 Hz."""
    floor = ct_floor(fs, fft)
    lo = floor * (1 + 1e-4)
    hi = max(min(1000.0, fs / 4.0), 1.05 * floor)
    rows = []
    for m in frames:
        f = rng.uniform(lo, hi, size=m)
        f[::5] = lo
        if at_floor:
            f[1::7] = 0.0
            f[3::11] = floor
        rows.append(f)
    return _rows(rows, frames)


def ct_dims(fft):
    return sorted({1, 2, fft // 8, fft // 4 + 1})


def check_cheaptrick(world, ref, fs, sizes, seed=0):
    """CheapTrick and CheapTrick + CodeSpectralEnvelope at every size in `sizes` against the reference's CheapTrick
    and CodeSpectralEnvelope.  Where the 500 Hz window does not fit, every f0 is above the floor.  The smallest
    size at which it fits also runs at q1 = -0.09."""
    x, lens, frames = _batch(fs, 1000 + seed)
    xb, tb = make(world, x), make(world, _time_rows(frames))
    t = _time_rows(frames)
    alt_q1 = min(s for s in POW2 if ct_defined(fs, s))
    worst = {}
    for fft in sizes:
        rng = np.random.default_rng([fs, fft, seed])
        f = ct_contours(rng, fs, fft, frames, at_floor=ct_defined(fs, fft))
        fb = make(world, f)
        for q1 in ((-0.15, -0.09) if fft == alt_q1 else (-0.15,)):
            opt = ct_option(fs, fft, q1)
            sp = world.cheaptrick(xb, fs, tb, fb, opt, x_lengths=lens, f0_lengths=frames)
            coded = {d: world.cheaptrick_coded(xb, fs, tb, fb, d, opt, x_lengths=lens, f0_lengths=frames)
                     for d in ct_dims(fft)}
            world.synchronize()
            sp = to_np(sp)
            assert sp.shape[2] == fft // 2 + 1
            _unwritten(sp, frames, f"CheapTrick fs {fs} fft {fft}")
            e = 0.0
            for u, m in enumerate(frames):
                want = ref.cheaptrick(x[u, :lens[u]], fs, t[u, :m], f[u, :m], opt)
                what = f"CheapTrick fs {fs} fft {fft} q1 {q1} utt {u}"
                assert_close(sp[u, :m], want, what)
                e = max(e, rel_err(sp[u, :m], want).max())
                for d, c in coded.items():
                    c = to_np(c)
                    assert_close_signed(c[u, :m], ref.code_spectral_envelope(want, fs, fft, d), f"coded {what} dims {d}")
                    assert not c[u, m:].any(), f"coded {what} dims {d}: padded frames were written"
            worst[(fs, fft)] = max(worst.get((fs, fft), 0.0), e)
    return worst


def check_cheaptrick_edomain(world, ref, fs, fft):
    """Below the size where the 500 Hz window fits: a frame at the floor or unvoiced is WORLD_B200_EDOMAIN at
    synchronize (plain and coded); the context keeps working, and with every f0 above the floor the call matches."""
    assert not ct_defined(fs, fft)
    x, lens, frames = _batch(fs, 1100)
    xb, tb = make(world, x), make(world, _time_rows(frames))
    opt = ct_option(fs, fft)
    rng = np.random.default_rng([fs, fft, 7])
    above = ct_contours(rng, fs, fft, frames, at_floor=False)
    for name, bad in (("unvoiced", 0.0), ("at the floor", ct_floor(fs, fft))):
        f = above.copy()
        f[1, frames[1] // 2] = bad
        for call in (lambda: world.cheaptrick(xb, fs, tb, make(world, f), opt, x_lengths=lens, f0_lengths=frames),
                     lambda: world.cheaptrick_coded(xb, fs, tb, make(world, f), 1, opt, x_lengths=lens,
                                                    f0_lengths=frames)):
            call()
            with pytest.raises(WorldError, match=r"error 4: device status 0x1: \[analysis window longer than fft_size"):
                world.synchronize()
            world.synchronize()                                 # the status word was cleared
    worst = check_cheaptrick(world, ref, fs, [fft], seed=1)
    return worst[(fs, fft)]


# ---------------------------------------------------------------- 3. D4C output size, plain and fused coded
def d4c_contours(rng, frames):
    """70-400 Hz with a fifth of the frames unvoiced and some below D4C's 47 Hz floor."""
    rows = []
    for m in frames:
        f = np.where(rng.uniform(size=m) < 0.8, rng.uniform(70.0, 400.0, size=m), 0.0)
        f[4::13] = 30.0
        rows.append(f)
    return _rows(rows, frames)


def check_d4c(world, ref, fs, sizes):
    """D4C and D4C + CodeAperiodicity at every output size in `sizes` against the reference's D4C and
    CodeAperiodicity."""
    x, lens, frames = _batch(fs, 1200)
    t, f = _time_rows(frames), d4c_contours(np.random.default_rng(fs), frames)
    xb, tb, fb = make(world, x), make(world, t), make(world, f)
    n_ap = ref.number_of_aperiodicities(fs)
    assert world.number_of_aperiodicities(fs) == n_ap > 0
    worst = {}
    for fft in sizes:
        ap = world.d4c(xb, fs, tb, fb, fft, x_lengths=lens, f0_lengths=frames)
        cap = world.d4c_coded(xb, fs, tb, fb, fft, x_lengths=lens, f0_lengths=frames)
        world.synchronize()
        ap, cap = to_np(ap), to_np(cap)
        assert ap.shape[2] == fft // 2 + 1 and cap.shape[2] == n_ap
        _unwritten(ap, frames, f"D4C fs {fs} fft {fft}")
        _unwritten(cap, frames, f"coded D4C fs {fs} fft {fft}")
        e = 0.0
        for u, m in enumerate(frames):
            want = ref.d4c(x[u, :lens[u]], fs, t[u, :m], f[u, :m], fft)
            assert_close(ap[u, :m], want, f"D4C fs {fs} fft {fft} utt {u}")
            assert_close_signed(cap[u, :m], ref.code_aperiodicity(want, fs, fft), f"coded D4C fs {fs} fft {fft} utt {u}")
            e = max(e, rel_err(ap[u, :m], want).max())
        worst[(fs, fft)] = e
    return worst


def check_d4c_tiny_sizes_refused(world):
    """fft_size 2 and 3 (defined in the reference, not served here) are WORLD_B200_EINVAL with a message that says so;
    the context keeps working."""
    fs = 16000
    x, lens, frames = _batch(fs, 1300)
    xb, tb = make(world, x), make(world, _time_rows(frames))
    fb = make(world, d4c_contours(np.random.default_rng(3), frames))
    for fft in (2, 3):
        for call in (world.d4c, world.d4c_coded):
            with pytest.raises(WorldError, match="error 3: D4C: fft_size must be at least 4"):
                call(xb, fs, tb, fb, fft, x_lengths=lens, f0_lengths=frames)
    world.d4c(xb, fs, tb, fb, 4, x_lengths=lens, f0_lengths=frames)
    world.synchronize()


# ---------------------------------------------------------------- 4. the codec
def check_codec(world, ref, fs, sizes, ap_sizes):
    """Code / DecodeSpectralEnvelope at every size in `sizes` and every dimension count of ct_dims, and Code /
    DecodeAperiodicity at every size in `ap_sizes`, against the reference, on ragged batches (the last utterance
    empty); fft_size / 4 + 2 dimensions is EINVAL."""
    n_ap = ref.number_of_aperiodicities(fs)
    assert world.number_of_aperiodicities(fs) == n_ap
    lens, F = [9, 4, 0], 9
    worst = {}
    for fft in sorted(set(sizes) | set(ap_sizes)):
        rng = np.random.default_rng([fs, fft])
        bins = fft // 2 + 1
        e = 0.0
        if fft in sizes:
            sp = np.exp(rng.normal(size=(3, F, bins)) * 3 - 8)
            for d in ct_dims(fft):
                a = to_np(world.code_spectral_envelope(make(world, sp), fs, fft, d, f0_lengths=lens))
                world.synchronize()
                back = np.zeros((3, F, d))
                for u in range(2):
                    want = ref.code_spectral_envelope(sp[u, :lens[u]], fs, fft, d)
                    assert_close_signed(a[u, :lens[u]], want, f"CodeSpectralEnvelope fs {fs} fft {fft} dims {d} utt {u}")
                    back[u, :lens[u]] = want
                _unwritten(a, lens, f"CodeSpectralEnvelope fs {fs} fft {fft} dims {d}")
                b = to_np(world.decode_spectral_envelope(make(world, back), fs, fft, d, f0_lengths=lens))
                world.synchronize()
                for u in range(2):
                    want = ref.decode_spectral_envelope(back[u, :lens[u]], fs, fft, d)
                    assert_close(b[u, :lens[u]], want, f"DecodeSpectralEnvelope fs {fs} fft {fft} dims {d} utt {u}")
                    e = max(e, rel_err(b[u, :lens[u]], want).max())
                _unwritten(b, lens, f"DecodeSpectralEnvelope fs {fs} fft {fft} dims {d}")
            with pytest.raises(WorldError, match="error 3: CodeSpectralEnvelope: number_of_dimensions"):
                world.code_spectral_envelope(make(world, sp), fs, fft, fft // 4 + 2, f0_lengths=lens)
        if fft in ap_sizes:
            ap = np.clip(rng.uniform(size=(3, F, bins)), 1e-3, 1 - 1e-12)
            ap[0, 2] = 1 - 1e-12                                 # an unvoiced frame
            coded = np.zeros((3, F, max(1, n_ap)))
            if n_ap > 0:
                a = to_np(world.code_aperiodicity(make(world, ap), fs, fft, f0_lengths=lens))
                world.synchronize()
                for u in range(2):
                    coded[u, :lens[u]] = ref.code_aperiodicity(ap[u, :lens[u]], fs, fft)
                    assert_close_signed(a[u, :lens[u]], coded[u, :lens[u]], f"CodeAperiodicity fs {fs} fft {fft} utt {u}")
                _unwritten(a, lens, f"CodeAperiodicity fs {fs} fft {fft}")
            b = to_np(world.decode_aperiodicity(make(world, coded), fs, fft, f0_lengths=lens))
            world.synchronize()
            for u in range(2):
                want = ref.decode_aperiodicity(coded[u, :lens[u]], fs, fft)
                assert_close(b[u, :lens[u]], want, f"DecodeAperiodicity fs {fs} fft {fft} utt {u}")
                e = max(e, rel_err(b[u, :lens[u]], want).max())
            _unwritten(b, lens, f"DecodeAperiodicity fs {fs} fft {fft}")
        worst[(fs, fft)] = e
    return worst


# ---------------------------------------------------------------- 5. Synthesis
def synthesis_lowest_f0(fs, fft):
    return fs // fft + 1.0                               # synthesis.cpp:362: integer division, then + 1.0


def synthesis_defined(fs, fft):
    """True when the 500 Hz pulses of unvoiced frames are at most 0.8 fft_size apart."""
    return fs / 500.0 <= 0.8 * fft


def pulse_intervals(f0, fs, fft, y_length):
    """The longest interval between two pulses of the reference's time base (synthesis.cpp:224-320, the noise_size
    of each pulse).  The contours of synthesis_rows end in two equal frames, so the linear extrapolation of the
    reference's interp1 beyond the last frame is np.interp's constant."""
    cf = np.where(f0 < synthesis_lowest_f0(fs, fft), 0.0, f0)
    cv = (cf != 0.0).astype(np.float64)
    cf, cv = np.append(cf, 2 * cf[-1] - cf[-2]), np.append(cv, 2 * cv[-1] - cv[-2])
    ct = np.arange(len(cf)) * (FP / 1000.0)
    t = np.arange(y_length) / float(fs)
    fi = np.where(np.interp(t, ct, cv) > 0.5, np.interp(t, ct, cf), 500.0)
    wrap = np.fmod(np.cumsum(2.0 * np.pi * fi / fs), 2.0 * np.pi)
    at = np.flatnonzero(np.abs(np.diff(wrap)) > np.pi)
    return int(np.diff(at).max()) if len(at) > 1 else 0


def synthesis_rows(rng, fs, fft, frames, between):
    """f0, envelope and aperiodicity rows.  Voiced f0 lies between 1.25 and 2.5 times the lowest f0, with runs of four
    unvoiced frames; the time base interpolates f0 towards 0 into an unvoiced run until the V/UV decision flips, which
    halves it, so voiced frames next to an unvoiced one lie between 2.5 and 3.1 times the lowest f0.  Each contour
    ends in two equal frames.  between: utterance 1 also gets runs of frames at and just above the lowest f0, below
    fs / fft_size + 1, inside voiced speech."""
    low, high = synthesis_lowest_f0(fs, fft), fs / fft + 1.0
    lo = 1.25 * low
    bins = fft // 2 + 1
    k = np.arange(bins) / bins
    f0s, sps, aps = [], [], []
    for u, m in enumerate(frames):
        f = rng.uniform(lo, 2.0 * lo, size=m)
        first = 52 if between and u == 1 else 7
        for s in range(first, m - 8, 17):
            f[s:s + 4] = 0.0
        voiced = f > 0
        edge = voiced & ~(np.append(voiced[1:], True) & np.insert(voiced[:-1], 0, True))
        f[edge] = rng.uniform(2.0 * lo, 2.5 * lo, size=int(edge.sum()))
        if between and u == 1:
            for i, v in enumerate((low, 0.5 * (low + high), np.nextafter(high, 0.0))):
                f[10 + 12 * i:18 + 12 * i] = v
        f[-1] = f[-2]
        f0s.append(f)
        sps.append(np.exp(-6.0 * k[None, :] + 0.3 * rng.normal(size=(m, 1))) * 1e-3)
        aps.append(np.clip(k[None, :] ** 2 + 0.05 * rng.uniform(size=(m, bins)), 1e-3, 1 - 1e-12))
    sp = np.ones((len(frames), max(frames), bins)); ap = np.ones_like(sp)
    for u, m in enumerate(frames):
        sp[u, :m] = sps[u]; ap[u, :m] = aps[u]
    return _rows(f0s, frames), sp, ap


def check_synthesis(world, ref, fs, sizes):
    """Synthesis at every size in `sizes` through its four forms: full rows; coded rows, equal to decode + full rows bit
    for bit; int16, equal to the quantised float64 call; the host call at nbit 0 and 16, equal to the device calls.
    Against the reference where it is defined with a margin, at 11.025 / 22.05 / 44.1 kHz with frames between the
    integer and the real lowest f0 (voiced in the reference).  fft_size 8192 is EINVAL for every form."""
    _, lens, frames = _batch(fs, 1400)
    ylens = [lens[0], int(lens[1] * 0.8), int(lens[2] * 1.2)]  # as long as the f0 grid, shorter, longer
    Y = max(ylens)
    n_ap = world.number_of_aperiodicities(fs)
    worst = {}
    for fft in sizes:
        rng = np.random.default_rng([fs, fft, 5])
        defined = synthesis_defined(fs, fft)
        between = defined and fs % fft != 0 and fs in (11025, 22050, 44100)
        f0, sp, ap = synthesis_rows(rng, fs, fft, frames, between)
        dims = min(fft // 4 + 1, 40)
        F, S, A = make(world, f0), make(world, sp), make(world, ap)
        y = world.synthesis(F, S, A, fft, FP, fs, Y, f0_lengths=frames, y_lengths=ylens)
        csp = world.code_spectral_envelope(S, fs, fft, dims, f0_lengths=frames)
        cap = world.code_aperiodicity(A, fs, fft, f0_lengths=frames) if n_ap > 0 else None
        dsp = world.decode_spectral_envelope(csp, fs, fft, dims, f0_lengths=frames)
        dap = world.decode_aperiodicity(cap if cap is not None else make(world, np.zeros((3, max(frames), 1))), fs, fft,
                                        f0_lengths=frames)
        two = world.synthesis(F, dsp, dap, fft, FP, fs, Y, f0_lengths=frames, y_lengths=ylens)
        yc = world.synthesis_coded(F, csp, cap, fft, FP, fs, Y, f0_lengths=frames, y_lengths=ylens)
        yq = world.synthesis_coded(F, csp, cap, fft, FP, fs, Y, f0_lengths=frames, y_lengths=ylens, dtype="int16")
        world.synchronize()
        y, two, yc, yq = to_np(y), to_np(two), to_np(yc), to_np(yq)
        what = f"Synthesis fs {fs} fft {fft}"
        assert np.isfinite(y).all() and np.isfinite(yc).all(), f"{what}: not finite"
        assert np.array_equal(yc, two), f"{what}: coded rows differ from decode + full rows"
        hcsp, hcap = to_np(csp), to_np(cap) if cap is not None else None
        for u, v in enumerate(ylens):
            assert not y[u, v:].any() and not yc[u, v:].any() and not yq[u, v:].any(), f"{what}: padding written"
            assert np.array_equal(yq[u, :v], quantise(yc[u, :v])), f"{what}: int16 differs from the quantised call"
            assert np.abs(y[u, :v]).max() > 0, f"{what}: utterance {u} is silent"
        for nbit, want in ((0, yc), (16, yq)):
            got = world.synthesis_coded_host(f0, hcsp, hcap, fft, FP, fs, Y, nbit=nbit, f0_lengths=frames,
                                             y_lengths=ylens)
            assert np.array_equal(got, want), f"{what}: host call at nbit {nbit} differs from the device call"
        if defined:
            e = 0.0
            for u, m in enumerate(frames):
                # the reference writes each interval of noise into fft_size samples: call it only where that fits
                iv = pulse_intervals(f0[u, :m], fs, fft, ylens[u])
                assert iv <= (fft if between and u == 1 else 0.8 * fft), f"{what} utt {u}: pulse interval {iv}"
                yr = ref.synthesis(f0[u, :m], sp[u, :m], ap[u, :m], fft, FP, fs, ylens[u])
                err = np.abs(y[u, :ylens[u]] - yr).max() / np.abs(yr).max()
                assert err <= 1e-9, f"{what} utt {u}: {err:.2e} of the peak"
                e = max(e, err)
            if between:
                low = synthesis_lowest_f0(fs, fft)
                assert ((f0[1] >= low) & (f0[1] < fs / fft + 1.0)).sum() == 24 and low < fs / fft + 1.0
            worst[(fs, fft)] = e
    # 8192 is beyond what every form serves
    F = make(world, np.full((1, 9), 200.0))
    S, A = make(world, np.ones((1, 9, 4097))), make(world, np.ones((1, 9, 4097)))
    csp = make(world, np.zeros((1, 9, 40)))
    cap = make(world, np.zeros((1, 9, max(1, n_ap)))) if n_ap > 0 else None
    for name, call in (
            ("synthesis", lambda: world.synthesis(F, S, A, 8192, FP, fs, 4000)),
            ("synthesis_coded", lambda: world.synthesis_coded(F, csp, cap, 8192, FP, fs, 4000)),
            ("synthesis_coded int16", lambda: world.synthesis_coded(F, csp, cap, 8192, FP, fs, 4000, dtype="int16")),
            ("synthesis_coded_host", lambda: world.synthesis_coded_host(to_np(F), to_np(csp), to_np(cap) if cap is not None
                                                                        else None, 8192, FP, fs, 4000))):
        with pytest.raises(WorldError, match="error 3: Synthesis: fft_size must be a power of two"):
            call()
    world.synchronize()
    return worst


# ---------------------------------------------------------------- 6. chains and the legacy API at another f0_floor
def check_chain_option(world, ref, fs, f0_floor, method):
    """analyze_batch, analyze_coded_batch, analyze_host and analyze_coded_host with CheapTrickOption.f0_floor changed
    (and fft_size from GetFFTSizeForCheapTrick) equal the stage calls at that option bit for bit; the legacy CheapTrick
    and D4C with that option match the reference."""
    x, lens, frames = _batch(fs, 1500)
    xb = make(world, x)
    ao = world.analysis_option(fs, method)
    ao.cheaptrick.f0_floor = f0_floor
    ao.cheaptrick.fft_size = world.lib.GetFFTSizeForCheapTrick(fs, C.byref(ao.cheaptrick))
    fft, dims = ao.cheaptrick.fft_size, 40
    assert fft != world.cheaptrick_option(fs).fft_size
    if method == F0_HARVEST:
        t, f0, fl = world.harvest(xb, fs, ao.harvest, x_lengths=lens)
    else:
        t, f0, fl = world.dio(xb, fs, ao.dio, x_lengths=lens)
        f0 = world.stonemask(xb, fs, t, f0, x_lengths=lens, f0_lengths=fl)
    assert fl == frames
    sp = world.cheaptrick(xb, fs, t, f0, ao.cheaptrick, x_lengths=lens, f0_lengths=fl)
    ap = world.d4c(xb, fs, t, f0, fft, ao.d4c, x_lengths=lens, f0_lengths=fl)
    csp = world.cheaptrick_coded(xb, fs, t, f0, dims, ao.cheaptrick, x_lengths=lens, f0_lengths=fl)
    cap = world.d4c_coded(xb, fs, t, f0, fft, ao.d4c, x_lengths=lens, f0_lengths=fl)
    chain = world.analyze_batch(xb, fs, ao, x_lengths=lens)
    coded = world.analyze_coded_batch(xb, 0, fs, ao, dims, x_lengths=lens)
    world.synchronize()
    host = world.analyze_host(x, fs, ao, x_lengths=lens)
    coded_host = world.analyze_coded_host(x, 0, fs, ao, dims, x_lengths=lens)
    want = [to_np(a) for a in (t, f0, sp, ap)]
    want_coded = [to_np(a) for a in (t, f0, csp, cap)]
    assert to_np(chain[2]).shape[2] == fft // 2 + 1
    for name, got, w in (("analyze_batch", chain, want), ("analyze_host", host, want),
                         ("analyze_coded_batch", coded, want_coded), ("analyze_coded_host", coded_host, want_coded)):
        assert list(got[4]) == fl
        for g, w_, part in zip(got[:4], w, ("time axis", "f0", "spectral rows", "aperiodicity rows")):
            g = to_np(g)
            for u, m in enumerate(fl):
                assert np.array_equal(g[u, :m], w_[u, :m]), \
                    f"{name} fs {fs} f0_floor {f0_floor}: {part} of utterance {u} differ from the stage calls"
    # the legacy entry points with that option, on utterance 0's f0
    lib = world.lib
    xu, m = np.ascontiguousarray(x[0, :lens[0]]), fl[0]
    tu, fu = np.ascontiguousarray(want[0][0, :m]), np.ascontiguousarray(want[1][0, :m])
    assert (fu > 0).sum() > 10
    bins = fft // 2 + 1
    lsp, lap = np.zeros((m, bins)), np.zeros((m, bins))
    rows = lambda a: (C.c_void_p * a.shape[0])(*[a[i].ctypes.data for i in range(a.shape[0])])
    lib.CheapTrick(xu.ctypes.data, len(xu), fs, tu.ctypes.data, fu.ctypes.data, m, C.byref(ao.cheaptrick), rows(lsp))
    d4 = D4COption(); lib.InitializeD4COption(C.byref(d4))
    lib.D4C(xu.ctypes.data, len(xu), fs, tu.ctypes.data, fu.ctypes.data, m, fft, C.byref(d4), rows(lap))
    spr = ref.cheaptrick(xu, fs, tu, fu, ao.cheaptrick)
    apr = ref.d4c(xu, fs, tu, fu, fft)
    assert_close(lsp, spr, f"legacy CheapTrick fs {fs} f0_floor {f0_floor}")
    assert_close(lap, apr, f"legacy D4C fs {fs} f0_floor {f0_floor}")
    assert_close(want[2][0, :m], spr, f"CheapTrick fs {fs} f0_floor {f0_floor}")
    return fft, max(rel_err(lsp, spr).max(), rel_err(lap, apr).max(), rel_err(want[2][0, :m], spr).max())


CHAIN_CASES = [(16000, 150.0, F0_DIO_STONEMASK), (16000, 150.0, F0_HARVEST), (16000, 40.0, F0_HARVEST),
               (44100, 40.0, F0_DIO_STONEMASK)]
