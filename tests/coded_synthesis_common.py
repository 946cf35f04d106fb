"""Checks of Synthesis from coded rows (world_b200_synthesis_coded_batch); the same assertions run against the host
emulation (CPU) and the CUDA library (-m gpu).  The main oracle is the two-step path of the same library
(decode_spectral_envelope + decode_aperiodicity + synthesis), which the call must equal bit for bit; the compiled
reference's DecodeSpectralEnvelope + DecodeAperiodicity + Synthesis is held to 1e-9 of the waveform peak, the bound of
every Synthesis test."""
import ctypes as C

import numpy as np

import test_parity_common as pc
from test_stage_paths import SMALL_BUDGET, _with_budget
from world_b200.api import F0_DIO_STONEMASK

EINVAL = 3


def analysed_rows(world, fs, fp, dims, seconds=0.9, seeds=(311, 312, 313)):
    """f0 and coded rows of synthetic speech from the library's own coded analysis (DIO + StoneMask at frame period fp),
    on a ragged batch: (f0, coded sp, coded ap, f0 lengths, x lengths), host arrays."""
    from synth import synth_batch
    n = int(seconds * fs)
    lens = [n - (u * fs) // 7 for u in range(len(seeds))]
    x = synth_batch(list(seeds), fs, n).numpy()
    ao = world.analysis_option(fs, F0_DIO_STONEMASK)
    ao.dio.frame_period = fp
    t, f0, csp, cap, fl = world.analyze_coded_batch(pc.make(world, x), 0, fs, ao, dims, x_lengths=lens)
    world.synchronize()
    return pc.to_np(f0), pc.to_np(csp), pc.to_np(cap), fl, lens


def perturb(rng, f0, csp, cap, fl, u):
    """Utterance u's rows made random around what analysis gave: noise on the cepstrum, band values anywhere in
    [-40, -0.01] dB, and every fifth frame fully unvoiced in the coded aperiodicity (mean > -0.5 dB)."""
    L = fl[u]
    csp[u, :L] += 0.05 * rng.normal(size=csp[u, :L].shape)
    if cap.shape[2] > 0:
        cap[u, :L] = rng.uniform(-40.0, -0.01, size=cap[u, :L].shape)
        cap[u, :L:5] = -0.2
    f0[u, :L] *= rng.uniform(0.7, 1.4)


def two_step(world, f0, csp, cap, fft, fp, fs, y_len, fl, yl):
    """decode_spectral_envelope + decode_aperiodicity + synthesis of the same library (device arrays in)."""
    dims = int(csp.shape[-1])
    sp = world.decode_spectral_envelope(csp, fs, fft, dims, f0_lengths=fl)
    if cap is None:   # no bands: the decoder reads nothing of its input
        cap = pc.make(world, np.zeros((f0.shape[0], f0.shape[1], 1)))
    ap = world.decode_aperiodicity(cap, fs, fft, f0_lengths=fl)
    y = world.synthesis(f0, sp, ap, fft, fp, fs, y_len, f0_lengths=fl, y_lengths=yl)
    world.synchronize()
    return pc.to_np(y)


def coded(world, f0, csp, cap, fft, fp, fs, y_len, fl, yl):
    y = world.synthesis_coded(f0, csp, cap, fft, fp, fs, y_len, f0_lengths=fl, y_lengths=yl)
    world.synchronize()
    return pc.to_np(y)


def ragged_y(fs, x_lens):
    """y lengths: the first utterance as analysed, the second shorter than its f0 grid implies, the third longer."""
    factors = (1.0, 0.7, 1.25)
    return [int(v * factors[u % 3]) for u, v in enumerate(x_lens)]


def assert_ref_close(y, yr, what):
    e = np.abs(y - yr).max() / max(np.abs(yr).max(), 1e-300)
    assert e <= 1e-9, f"{what}: {e:.2e} of the peak"
    return e


def check_equals_two_step(world, fs, fp, dims, seed=0):
    """Every output row equals the two-step path bit for bit: a ragged batch (f0 and y lengths differ per utterance,
    y_length shorter and longer than the f0 grid implies), rows from analysis (utterance 0) and perturbed random rows
    with fully unvoiced frames (utterances 1, 2)."""
    f0, csp, cap, fl, lens = analysed_rows(world, fs, fp, dims)
    rng = np.random.default_rng(1000 * fs + 10 * int(fp * 2) + dims + seed)
    for u in (1, 2):
        perturb(rng, f0, csp, cap, fl, u)
    n_ap = world.number_of_aperiodicities(fs)
    assert (f0[0, :fl[0]] > 0).sum() > 10 and (f0[0, :fl[0]] == 0).sum() > 5
    if n_ap > 0:
        assert (cap[1, :fl[1]].mean(axis=1) > -0.5).sum() >= fl[1] // 5
    fft = world.cheaptrick_option(fs).fft_size
    yl = ragged_y(fs, lens)
    Y = max(yl)
    F, S = pc.make(world, f0), pc.make(world, csp)
    A = pc.make(world, cap) if n_ap > 0 else None
    want = two_step(world, F, S, A, fft, fp, fs, Y, fl, yl)
    got = coded(world, F, S, A, fft, fp, fs, Y, fl, yl)
    assert got.shape == want.shape
    for u in range(len(fl)):
        assert np.abs(want[u, :yl[u]]).max() > 1e-4, f"utterance {u} is silent"
        assert np.array_equal(got[u], want[u]), f"fs {fs} fp {fp} dims {dims}: utterance {u} differs from the two-step path"


def check_vs_reference(world, ref, golden):
    """The golden fixture's coded rows and three synthetic utterances' coded rows through the reference's
    DecodeSpectralEnvelope + DecodeAperiodicity + Synthesis: within 1e-9 of the waveform peak."""
    fs, fft, dims = int(golden["fs"]), int(golden["fft_size"]), int(golden["coded_dims"])
    f0, csp, cap = golden["f0_stonemask"], golden["coded_sp"], golden["coded_ap"]
    n = len(golden["pcm"])
    y = coded(world, pc.make(world, f0[None]), pc.make(world, csp[None]), pc.make(world, cap[None]), fft, 5.0, fs, n,
              None, None)
    yr = ref.synthesis(f0, ref.decode_spectral_envelope(csp, fs, fft, dims), ref.decode_aperiodicity(cap, fs, fft), fft,
                       5.0, fs, n)
    worst = assert_ref_close(y[0], yr, "golden coded rows")
    fs, fp, dims = 16000, 5.0, 60
    f0, csp, cap, fl, lens = analysed_rows(world, fs, fp, dims, seeds=(321, 322, 323))
    fft = world.cheaptrick_option(fs).fft_size
    yl = ragged_y(fs, lens)
    y = coded(world, pc.make(world, f0), pc.make(world, csp), pc.make(world, cap), fft, fp, fs, max(yl), fl, yl)
    for u in range(3):
        L = fl[u]
        yr = ref.synthesis(f0[u, :L], ref.decode_spectral_envelope(csp[u, :L], fs, fft, dims),
                           ref.decode_aperiodicity(cap[u, :L], fs, fft), fft, fp, fs, yl[u])
        worst = max(worst, assert_ref_close(y[u, :yl[u]], yr, f"synthetic utterance {u}"))
    return worst


def check_no_bands(world, ref, fs=8000):
    """Below 12 kHz: coded_aperiodicity None, equal to the two-step path (which decodes zero bands) and within the
    reference bound."""
    fp, dims = 5.0, 40
    assert world.number_of_aperiodicities(fs) == 0
    f0, csp, _, fl, lens = analysed_rows(world, fs, fp, dims, seeds=(331, 332, 333))
    fft = world.cheaptrick_option(fs).fft_size
    yl = ragged_y(fs, lens)
    F, S = pc.make(world, f0), pc.make(world, csp)
    want = two_step(world, F, S, None, fft, fp, fs, max(yl), fl, yl)
    got = coded(world, F, S, None, fft, fp, fs, max(yl), fl, yl)
    assert np.array_equal(got, want)
    worst = 0.0
    for u in range(3):
        L = fl[u]
        yr = ref.synthesis(f0[u, :L], ref.decode_spectral_envelope(csp[u, :L], fs, fft, dims),
                           ref.decode_aperiodicity(np.zeros((L, 1)), fs, fft), fft, fp, fs, yl[u])
        worst = max(worst, assert_ref_close(got[u, :yl[u]], yr, f"8 kHz utterance {u}"))
    return worst


def envelope_rows(world, rng, fs, fft, dims, flens, L, f0_hz=None):
    """f0 and coded rows of smooth random envelopes / aperiodicities coded by the library's own codec."""
    n_utt, bins = len(flens), fft // 2 + 1
    f0 = np.zeros((n_utt, L)); sp = np.ones((n_utt, L, bins)); ap = np.ones((n_utt, L, bins))
    k = np.arange(bins) / bins
    for u, m in enumerate(flens):
        f0[u, :m] = np.where(rng.uniform(size=m) < 0.85, rng.uniform(90.0, 300.0) * (1 + 0.2 * np.sin(np.arange(m) / 30.0)), 0.0)
        sp[u, :m] = np.exp(-6.0 * k[None, :] + 0.3 * rng.normal(size=(m, 1))) * 1e-3
        ap[u, :m] = np.clip(k[None, :] ** 2 + 0.05 * rng.uniform(size=(m, bins)), 1e-3, 1 - 1e-12)
    if f0_hz is not None:
        for u, hz in f0_hz.items():
            f0[u, :flens[u]] = hz
    csp = world.code_spectral_envelope(pc.make(world, sp), fs, fft, dims, f0_lengths=flens)
    cap = world.code_aperiodicity(pc.make(world, ap), fs, fft, f0_lengths=flens)
    world.synchronize()
    return pc.make(world, f0), csp, cap


def check_small_budget(world):
    """At the smallest scratch budget the call runs in several chunks, the last one shorter, and gives the one-chunk
    result bit for bit.  Per utterance (2 s at 16 kHz, fft 1024): the full-row call's 20,878,496 B (see
    test_stage_paths.check_chunks_synthesis) plus 401 frames * 513 bins * 16 B of decoded rows = 24,169,904 B, so two
    utterances per 64 MB pass: 7 utterances -> passes of 2, 2, 2, 1.  Each pass launches the same kernels (no pass has
    more than 1,200 pulses per second), so the pass count is the ratio of the launch counts."""
    fs, n_utt, secs, fft, dims = 16000, 7, 2.0, 1024, 40
    n = int(secs * fs)
    ylens = [n - 1337 * u for u in range(n_utt)]
    L = int(secs * 200) + 1
    flens = [L - 7 * u for u in range(n_utt)]
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs, launches = [], []
        for w in (world, small):
            f0, csp, cap = envelope_rows(w, np.random.default_rng(23), fs, fft, dims, flens, L)
            before = w.launch_count()
            outs.append(coded(w, f0, csp, cap, fft, 5.0, fs, n, flens, ylens))
            launches.append(w.launch_count() - before)
    finally:
        small.close()
    assert launches[1] == 4 * launches[0], f"launches: {launches[0]} in one pass, {launches[1]} at the small budget"
    assert outs[0].shape == outs[1].shape and np.array_equal(outs[0], outs[1]), "chunked result differs"
    assert np.abs(outs[1][n_utt - 1]).max() > 1e-4


def check_high_f0(world):
    """One utterance at 2 kHz (beyond the 1,200 pulses per second the arrays are first laid out for) forces the relaid
    pass (one more time-base launch); the result equals the two-step path."""
    fs, fft, dims, secs = 16000, 1024, 40, 1.0
    rng = np.random.default_rng(29)
    n = int(secs * fs)
    L = int(secs * 200) + 1
    flens = [L, L - 11, L - 23]
    ylens = [n, n - 901, n - 1802]
    f0, csp, cap = envelope_rows(world, rng, fs, fft, dims, flens, L, f0_hz={1: 2000.0})
    want = two_step(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens)
    before = world.launch_count()
    got = coded(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens)
    relaid = world.launch_count() - before
    low = f0.clone() if hasattr(f0, "clone") else f0.copy()
    low[1] = low[0]
    before = world.launch_count()
    coded(world, low, csp, cap, fft, 5.0, fs, n, flens, ylens)
    assert relaid == world.launch_count() - before + 1, "the 2 kHz utterance did not take the relaid pass"
    assert np.array_equal(got, want), "f0 above 1.2 kHz: differs from the two-step path"


def _ptr(a):
    if a is None:
        return None
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def check_invalid(world):
    """Every bad argument is EINVAL before any work: nothing is launched and the output keeps its sentinel; the context
    keeps working."""
    fs, fp, fft, dims = 16000, 5.0, 1024, 40
    rng = np.random.default_rng(31)
    L, n, Y = 81, 3, 6400
    flens, ylens = [L, L - 5, L - 9], [Y, Y - 100, Y - 333]
    f0, csp, cap = envelope_rows(world, rng, fs, fft, dims, flens, L)
    y = pc.make(world, np.full((n, Y), -7.0))
    lib = world.lib

    def call(fft_size=fft, d=dims, ap=cap, fl=flens, yl=ylens, f0_stride=L, y_stride=Y, rate=fs, sp=csp):
        world._use_current_stream()
        before = world.launch_count()
        rc = lib.world_b200_synthesis_coded_batch(world._h, _ptr(f0), (C.c_int * n)(*fl), n, f0_stride, _ptr(sp), d,
                                                  _ptr(ap), fft_size, fp, rate, (C.c_int * n)(*yl), y_stride, _ptr(y))
        world.synchronize()
        return rc, world.launch_count() - before

    cases = [
        ("fft_size 8192", dict(fft_size=8192)),
        ("fft_size 1000", dict(fft_size=1000)),
        ("fft_size 8", dict(fft_size=8)),
        ("number_of_dimensions 0", dict(d=0)),
        ("number_of_dimensions fft_size/2 + 1", dict(d=fft // 2 + 1)),
        ("NULL coded_aperiodicity at 16 kHz", dict(ap=None)),
        ("NULL coded_spectral_envelope", dict(sp=None)),
        ("f0 length beyond its row", dict(fl=[L, L + 1, L - 9])),
        ("f0 length 1", dict(fl=[L, 1, L - 9])),
        ("y length beyond its row", dict(yl=[Y, Y + 1, Y - 333])),
        ("y length 1", dict(yl=[Y, Y - 100, 1])),
    ]
    for what, kw in cases:
        rc, launched = call(**kw)
        assert rc == EINVAL, f"{what}: returned {rc}"
        assert launched == 0, f"{what}: {launched} kernels launched"
        assert (pc.to_np(y) == -7.0).all(), f"{what}: the output was written"
    rc, launched = call()
    assert rc == 0 and launched > 0
    assert all(not (pc.to_np(y)[u, :ylens[u]] == -7.0).any() for u in range(n))
    import pytest
    from world_b200.api import WorldError
    with pytest.raises(WorldError, match="error 3: .*number_of_dimensions"):
        world.synthesis_coded(f0, pc.make(world, np.zeros((n, L, fft // 2 + 1))), cap, fft, fp, fs, Y,
                              f0_lengths=flens, y_lengths=ylens)
