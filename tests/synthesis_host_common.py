"""Checks of Synthesis from coded rows to 16-bit PCM (world_b200_synthesis_coded_batch_pcm16) and of the pipelined host
call (world_b200_synthesis_coded_host); the same assertions run against the host emulation (CPU) and the CUDA library
(-m gpu).  The oracle is the float64 coded call of the same library, quantised as wavwrite quantises:
trunc(y * 32767) clamped to [-32768, 32767], which every PCM sample must equal bit for bit."""
import ctypes as C
import re

import numpy as np

import coded_synthesis_common as cs
import test_parity_common as pc
from test_stage_paths import SMALL_BUDGET, _with_budget

EINVAL = 3


def quantise(y):
    """wavwrite's rule: (int)(y * 32767) toward zero, clamped (beyond the int range: saturated by sign)."""
    return np.clip(np.trunc(np.asarray(y) * 32767), -32768, 32767).astype(np.int16)


def _ptr(a):
    return cs._ptr(a)


def pcm16_into(world, y, f0, csp, cap, fft, fp, fs, fl, yl):
    """world_b200_synthesis_coded_batch_pcm16 into a caller's int16 array y (kept as given where not written)."""
    n, L = f0.shape[0], f0.shape[1]
    fla = (C.c_int * n)(*fl) if fl is not None else None
    yla = (C.c_int * n)(*yl) if yl is not None else None
    world._use_current_stream()
    rc = world.lib.world_b200_synthesis_coded_batch_pcm16(world._h, _ptr(f0), fla, n, L, _ptr(csp), int(csp.shape[-1]),
                                                          _ptr(cap), fft, fp, fs, yla, int(y.shape[1]), _ptr(y))
    world.synchronize()
    return rc


def device_pair(world, f0, csp, cap, fft, fp, fs, y_len, fl, yl):
    """(float64 waveform, int16 PCM) of the device calls, host arrays."""
    yd = world.synthesis_coded(f0, csp, cap, fft, fp, fs, y_len, f0_lengths=fl, y_lengths=yl)
    yq = world.synthesis_coded(f0, csp, cap, fft, fp, fs, y_len, f0_lengths=fl, y_lengths=yl, dtype="int16")
    world.synchronize()
    return pc.to_np(yd), pc.to_np(yq)


def assert_quantised(yq, yd, yl, what):
    assert yq.dtype == np.int16
    for u in range(len(yl)):
        want = quantise(yd[u, :yl[u]])
        bad = np.flatnonzero(yq[u, :yl[u]] != want)
        assert bad.size == 0, f"{what}: utterance {u}, {bad.size} samples differ (first {bad[0]}: " \
                              f"{yq[u, bad[0]]} vs {want[bad[0]]} from {yd[u, bad[0]]!r})"


def wavwrite_pcm(world, y, fs, path):
    """The data chunk the library's own wavwrite() writes for the float64 samples y."""
    y = np.ascontiguousarray(y, dtype=np.float64)
    world.lib.wavwrite(y.ctypes.data, len(y), fs, 16, str(path).encode())
    data = open(path, "rb").read()
    assert data[36:40] == b"data"
    return np.frombuffer(data[44:], dtype="<i2")


def check_pcm_equals_quantised(world, fs, fp, dims, tmp_path):
    """The int16 device call equals the quantised float64 call on a ragged batch of analysed (utterance 0) and perturbed
    rows, and equals the wavwrite data chunk of utterance 0; padding prefilled with a sentinel stays untouched."""
    f0, csp, cap, fl, lens = cs.analysed_rows(world, fs, fp, dims)
    rng = np.random.default_rng(2000 * fs + 10 * int(fp * 2) + dims)
    for u in (1, 2):
        cs.perturb(rng, f0, csp, cap, fl, u)
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    Y = max(yl)
    F, S = pc.make(world, f0), pc.make(world, csp)
    A = pc.make(world, cap) if world.number_of_aperiodicities(fs) > 0 else None
    yd, yq = device_pair(world, F, S, A, fft, fp, fs, Y, fl, yl)
    for u in range(len(yl)):
        assert np.abs(yq[u, :yl[u]]).max() > 30, f"utterance {u} is silent"
    assert_quantised(yq, yd, yl, f"fs {fs} fp {fp} dims {dims}")
    assert np.array_equal(wavwrite_pcm(world, yd[0, :yl[0]], fs, tmp_path / "u0.wav"), yq[0, :yl[0]]), \
        "utterance 0 differs from the library's wavwrite"
    y = pc.make(world, np.full((len(yl), Y), -12345), dtype=np.int16)
    assert pcm16_into(world, y, F, S, A, fft, fp, fs, fl, yl) == 0
    y = pc.to_np(y)
    for u in range(len(yl)):
        assert np.array_equal(y[u, :yl[u]], yq[u, :yl[u]])
        assert (y[u, yl[u]:] == -12345).all(), f"utterance {u}: padding was written"


def check_pcm_clips(world):
    """An envelope scaled up clips in both directions: by exp(6) the samples leave [-1, 1] (the defined range of the
    cast), by exp(50) they leave the int range, where both the kernel and the numpy rule saturate by sign."""
    fs, fp, dims = 16000, 5.0, 40
    f0, csp, cap, fl, lens = cs.analysed_rows(world, fs, fp, dims, seconds=0.5, seeds=(351, 352, 353))
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    F, A = pc.make(world, f0), pc.make(world, cap)
    for add, beyond_int in ((6.0, False), (50.0, True)):
        c = csp.copy()
        c[..., 0] += add
        yd, yq = device_pair(world, F, pc.make(world, c), A, fft, fp, fs, max(yl), fl, yl)
        assert_quantised(yq, yd, yl, f"envelope scaled by exp({add:g})")
        q = np.concatenate([yq[u, :yl[u]] for u in range(len(yl))])
        assert (q == 32767).any() and (q == -32768).any(), f"exp({add:g}): no clipping in both directions"
        peak = np.abs(yd).max() * 32767
        assert (peak >= 2.0 ** 31) == beyond_int, f"peak {peak:.3g} of the quantiser's input"


def check_host_equals_device(world, fs=16000, fp=5.0, dims=60):
    """synthesis_coded_host: nbit 0 equals the float64 device call and nbit 16 the int16 one, bit for bit; padded
    samples are 0."""
    f0, csp, cap, fl, lens = cs.analysed_rows(world, fs, fp, dims, seeds=(361, 362, 363))
    rng = np.random.default_rng(47)
    cs.perturb(rng, f0, csp, cap, fl, 2)
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    Y = max(yl)
    yd, yq = device_pair(world, pc.make(world, f0), pc.make(world, csp), pc.make(world, cap), fft, fp, fs, Y, fl, yl)
    for nbit, want in ((0, yd), (16, yq)):
        out = np.full((len(yl), Y), 77, dtype=want.dtype)   # whole rows are written back
        got = world.synthesis_coded_host(f0, csp, cap, fft, fp, fs, Y, nbit=nbit, f0_lengths=fl, y_lengths=yl, out=out)
        assert got.dtype == want.dtype and got.shape == want.shape
        for u in range(len(yl)):
            assert np.array_equal(got[u, :yl[u]], want[u, :yl[u]]), f"nbit {nbit}: utterance {u} differs from the device"
            assert (got[u, yl[u]:] == 0).all(), f"nbit {nbit}: utterance {u}: padded samples are not 0"
    return yd, yq


def trace_chunks(text):
    """(chunks, ring) of the last synthesis line WB_HOST_TRACE printed."""
    found = re.findall(r"\[wb trace\] synthesis chunk \d+ chunks (\d+) ring (\d+)", text)
    assert found, f"no synthesis trace line in:\n{text}"
    return tuple(int(v) for v in found[-1])


def check_pipeline_chunks(world, capfd, monkeypatch):
    """At the smallest scratch budget the host call runs in at least 3 chunks (one pass of synthesis_run each: two
    utterances of 2 s, see coded_synthesis_common.check_small_budget) and wraps its output ring; its output equals the
    default budget's, which runs in one chunk."""
    fs, n_utt, secs, fft, dims = 16000, 7, 2.0, 1024, 40
    n = int(secs * fs)
    ylens = [n - 1337 * u for u in range(n_utt)]
    L = int(secs * 200) + 1
    flens = [L - 7 * u for u in range(n_utt)]
    f0, csp, cap = cs.envelope_rows(world, np.random.default_rng(53), fs, fft, dims, flens, L)
    f0, csp, cap = pc.to_np(f0), pc.to_np(csp), pc.to_np(cap)
    monkeypatch.setenv("WB_HOST_TRACE", "1")
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs, shape = [], []
        for w in (world, small):
            capfd.readouterr()
            outs.append(w.synthesis_coded_host(f0, csp, cap, fft, 5.0, fs, n, nbit=16, f0_lengths=flens,
                                               y_lengths=ylens))
            shape.append(trace_chunks(capfd.readouterr().err))
    finally:
        small.close()
        monkeypatch.delenv("WB_HOST_TRACE")
    (chunks0, _), (chunks, ring) = shape
    assert chunks0 == 1, f"default budget: {chunks0} chunks"
    assert chunks >= 3 and chunks > ring, f"small budget: {chunks} chunks over a ring of {ring}"
    assert np.array_equal(outs[0], outs[1]), "chunked result differs"
    assert np.abs(outs[1][n_utt - 1, :ylens[-1]]).max() > 30
    assert (outs[1][n_utt - 1, ylens[-1]:] == 0).all()


def check_host_high_f0(world):
    """A 2 kHz utterance (the relaid pass of synthesis_run) through the host call, nbit 16: equal to the quantised
    two-step path and to the int16 device call."""
    fs, fft, dims, secs = 16000, 1024, 40, 1.0
    n = int(secs * fs)
    L = int(secs * 200) + 1
    flens = [L, L - 11, L - 23]
    ylens = [n, n - 901, n - 1802]
    f0, csp, cap = cs.envelope_rows(world, np.random.default_rng(59), fs, fft, dims, flens, L, f0_hz={1: 2000.0})
    want = cs.two_step(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens)
    _, yq = device_pair(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens)
    got = world.synthesis_coded_host(pc.to_np(f0), pc.to_np(csp), pc.to_np(cap), fft, 5.0, fs, n, nbit=16,
                                     f0_lengths=flens, y_lengths=ylens)
    assert_quantised(got, want, ylens, "2 kHz utterance, host call")
    assert np.array_equal(got, yq)


def check_vs_reference(world, ref, golden):
    """The golden fixture's coded rows and three synthetic utterances through the reference's DecodeSpectralEnvelope +
    DecodeAperiodicity + Synthesis, quantised by the same rule: the int16 device call and the host call are within
    1 LSB (a sample within 1e-9 of the peak of the reference may cross a quantisation step)."""
    def close(got, yr, what):
        d = np.abs(got.astype(np.int32) - quantise(yr).astype(np.int32)).max()
        assert d <= 1, f"{what}: {d} LSB from the reference"
        return int(d)

    fs, fft, dims = int(golden["fs"]), int(golden["fft_size"]), int(golden["coded_dims"])
    f0, csp, cap = golden["f0_stonemask"], golden["coded_sp"], golden["coded_ap"]
    n = len(golden["pcm"])
    yr = ref.synthesis(f0, ref.decode_spectral_envelope(csp, fs, fft, dims), ref.decode_aperiodicity(cap, fs, fft), fft,
                       5.0, fs, n)
    y = world.synthesis_coded(pc.make(world, f0[None]), pc.make(world, csp[None]), pc.make(world, cap[None]), fft, 5.0,
                              fs, n, dtype="int16")
    world.synchronize()
    worst = close(pc.to_np(y)[0], yr, "golden coded rows")
    yh = world.synthesis_coded_host(f0[None], csp[None], cap[None], fft, 5.0, fs, n)
    assert np.array_equal(yh, pc.to_np(y))
    fs, fp, dims = 16000, 5.0, 60
    f0, csp, cap, fl, lens = cs.analysed_rows(world, fs, fp, dims, seeds=(321, 322, 323))
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    y = world.synthesis_coded_host(f0, csp, cap, fft, fp, fs, max(yl), f0_lengths=fl, y_lengths=yl)
    for u in range(3):
        L = fl[u]
        yr = ref.synthesis(f0[u, :L], ref.decode_spectral_envelope(csp[u, :L], fs, fft, dims),
                           ref.decode_aperiodicity(cap[u, :L], fs, fft), fft, fp, fs, yl[u])
        worst = max(worst, close(y[u, :yl[u]], yr, f"synthetic utterance {u}"))
    return worst


def check_no_bands(world, fs=8000):
    """Below 12 kHz coded_aperiodicity is None in both calls; host nbit 0 / 16 equal the device calls."""
    fp, dims = 5.0, 40
    assert world.number_of_aperiodicities(fs) == 0
    f0, csp, _, fl, lens = cs.analysed_rows(world, fs, fp, dims, seeds=(371, 372, 373))
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    yd, yq = device_pair(world, pc.make(world, f0), pc.make(world, csp), None, fft, fp, fs, max(yl), fl, yl)
    assert_quantised(yq, yd, yl, "8 kHz")
    for nbit, want in ((0, yd), (16, yq)):
        got = world.synthesis_coded_host(f0, csp, None, fft, fp, fs, max(yl), nbit=nbit, f0_lengths=fl, y_lengths=yl)
        assert np.array_equal(got, want), f"8 kHz, nbit {nbit}: host differs from the device"


def check_invalid(world):
    """n_utts 0 returns 0; bad nbit, a NULL coded aperiodicity where fs has bands and bad lengths are EINVAL before any
    work: nothing is launched and the output keeps its sentinel (host call and int16 device call)."""
    fs, fp, fft, dims = 16000, 5.0, 1024, 40
    rng = np.random.default_rng(61)
    L, n, Y = 81, 3, 6400
    flens, ylens = [L, L - 5, L - 9], [Y, Y - 100, Y - 333]
    f0, csp, cap = cs.envelope_rows(world, rng, fs, fft, dims, flens, L)
    hf0, hsp, hap = pc.to_np(f0), pc.to_np(csp), pc.to_np(cap)
    lib = world.lib

    def host(nbit=16, ap=hap, fl=flens, yl=ylens, n_utts=n, fft_size=fft):
        y = np.full((n, Y), 99 if nbit == 16 else 99.0, dtype=np.int16 if nbit == 16 else np.float64)
        before = world.launch_count()
        rc = lib.world_b200_synthesis_coded_host(world._h, _ptr(hf0), (C.c_int * n)(*fl), n_utts, L, _ptr(hsp), dims,
                                                 _ptr(ap), fft_size, fp, fs, (C.c_int * n)(*yl), Y, nbit, _ptr(y))
        return rc, world.launch_count() - before, (y == 99).all()

    def device(ap=cap, fl=flens, yl=ylens, n_utts=n, fft_size=fft):
        y = pc.make(world, np.full((n, Y), 99), dtype=np.int16)
        world._use_current_stream()
        before = world.launch_count()
        rc = lib.world_b200_synthesis_coded_batch_pcm16(world._h, _ptr(f0), (C.c_int * n)(*fl), n_utts, L, _ptr(csp),
                                                        dims, _ptr(ap), fft_size, fp, fs, (C.c_int * n)(*yl), Y,
                                                        _ptr(y))
        world.synchronize()
        return rc, world.launch_count() - before, (pc.to_np(y) == 99).all()

    rc, launched, kept = host(n_utts=0)
    assert rc == 0 and launched == 0 and kept, "n_utts 0"
    rc, launched, kept = device(n_utts=0)
    assert rc == 0 and launched == 0 and kept, "n_utts 0 (device)"
    cases = [
        ("nbit 8", dict(nbit=8)),
        ("nbit 24", dict(nbit=24)),
        ("nbit 32", dict(nbit=32)),
        ("fft_size 1000", dict(fft_size=1000)),
        ("NULL coded_aperiodicity at 16 kHz", dict(ap=None)),
        ("f0 length beyond its row", dict(fl=[L, L + 1, L - 9])),
        ("f0 length 1", dict(fl=[L, 1, L - 9])),
        ("y length beyond its row", dict(yl=[Y, Y + 1, Y - 333])),
        ("y length 1 in the last utterance", dict(yl=[Y, Y - 100, 1])),
    ]
    for what, kw in cases:
        rc, launched, kept = host(**kw)
        assert rc == EINVAL, f"host, {what}: returned {rc}"
        assert launched == 0 and kept, f"host, {what}: {launched} kernels launched, output kept: {kept}"
        if "nbit" not in kw:
            rc, launched, kept = device(**kw)
            assert rc == EINVAL and launched == 0 and kept, f"device, {what}: rc {rc}, {launched} launched"
    rc, launched, kept = host()
    assert rc == 0 and launched > 0 and not kept
    import pytest
    from world_b200.api import WorldError
    with pytest.raises(WorldError, match="error 3: .*nbit"):
        world.synthesis_coded_host(hf0, hsp, hap, fft, fp, fs, Y, nbit=8, f0_lengths=flens, y_lengths=ylens)
    with pytest.raises(ValueError):
        world.synthesis_coded(f0, csp, cap, fft, fp, fs, Y, f0_lengths=flens, y_lengths=ylens, dtype="int32")
