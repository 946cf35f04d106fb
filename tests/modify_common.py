"""Checks of F0 scaling and formant shift (world_b200_modify_batch and the modified synthesis calls); the same
assertions run against the host emulation (CPU) and the CUDA library (-m gpu).

The oracle of the modification is the reference demo's ParameterModification (test/test.cpp:221-258) restated below:
the reference's own interp1, from the compiled reference library, and the host's libm log / exp (Python's math).  The
modified synthesis calls are held bit for bit to the step-by-step chain of the same library (decode, modify, decode,
synthesis), and the reference demo itself is run on the fixture and compared with the library's chain."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

import test_parity_common as pc
import coded_synthesis_common as cs
from test_stage_paths import SMALL_BUDGET, _with_budget
from world_b200.api import F0_DIO_STONEMASK

EINVAL = 3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DEMO = os.path.join(ROOT, "oracle", "_ref", "ref_demo")
SCALES = (0.5, 1.0, 1.5, 2.0)


def ratios_for(fft):
    """The per-utterance ratios of one call: shrink and stretch, 1.0, and the smallest ratio that keeps
    c = (int)(fft / 2.0 * ratio) == 1 (fft / 2.0 * (2 / fft) is exactly 1.0)."""
    return (0.5, 0.83, 1.0, 1.2, 2.0, 3.7, 2.0 / fft)


# ---- the reference semantics, restated ------------------------------------------------------------------------------
def ref_interp1(ref):
    fn = ref.lib.interp1
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    return fn


def _exp(v):
    """libm's exp, which gives inf where Python's raises (extrapolated bins that the tail rule then overwrites)."""
    try:
        return math.exp(v)
    except OverflowError:
        return math.inf


def ref_modify(ref, f0, sp, fs, fft, shift, ratio):
    """ParameterModification of test.cpp:221-258 for one utterance's frames: f0 [L], sp [L][fft/2+1] (host arrays,
    returned changed copies; shift / ratio None skip that half)."""
    f0, sp = np.array(f0, dtype=np.float64), np.array(sp, dtype=np.float64)
    if shift is not None:
        for i in range(len(f0)):
            f0[i] = f0[i] * shift
    if ratio is None:
        return f0, sp
    interp1 = ref_interp1(ref)
    half = fft // 2
    bins = half + 1
    x = (C.c_double * bins)(*[ratio * i / fft * fs for i in range(bins)])
    xi = (C.c_double * bins)(*[float(i) / fft * fs for i in range(bins)])
    y, out = (C.c_double * bins)(), (C.c_double * bins)()
    for i in range(sp.shape[0]):
        for j in range(bins):
            y[j] = math.log(sp[i, j])
        interp1(C.addressof(x), C.addressof(y), bins, C.addressof(xi), bins, C.addressof(out))
        row = [_exp(out[j]) for j in range(bins)]
        if ratio < 1.0:
            c = int(fft / 2.0 * ratio)
            row[c:] = [row[c - 1]] * (bins - c)
        sp[i] = row
    return f0, sp


# ---- rows ------------------------------------------------------------------------------------------------------------
def analysed_full_rows(world, fs, fft, seconds=0.35, seeds=(411, 412, 413)):
    """f0 and envelope rows of a ragged batch of synthetic speech from the library's own analysis (DIO + StoneMask,
    CheapTrick at fft), tiled to seven utterances: (f0 [7, L], sp [7, L, fft/2+1], f0 lengths), host arrays."""
    from synth import synth_batch
    n = int(seconds * fs)
    lens = [n - (u * fs) // 20 for u in range(len(seeds))]
    x = synth_batch(list(seeds), fs, n).numpy()
    ao = world.analysis_option(fs, F0_DIO_STONEMASK)
    ao.cheaptrick.fft_size = fft
    ao.cheaptrick.f0_floor = max(ao.cheaptrick.f0_floor, 3.0 * fs / (fft - 3.0) + 1.0)
    t, f0, sp, ap, fl = world.analyze_batch(pc.make(world, x), fs, ao, x_lengths=lens, aperiodicity=None)
    world.synchronize()
    f0, sp = pc.to_np(f0), pc.to_np(sp)
    pick = [u % len(seeds) for u in range(7)]
    return f0[pick].copy(), sp[pick].copy(), [fl[u] for u in pick]


def modify(world, f0, sp, fs, fft, scales, ratios, fl):
    F, S = pc.make(world, f0.copy()), pc.make(world, sp.copy())   # copies: make() may hand back the numpy array itself
    world.modify(F, S, fs, fft, f0_scale=scales, spectral_ratio=ratios, f0_lengths=fl)
    world.synchronize()
    return pc.to_np(F), pc.to_np(S)


def rel_worst(got, want):
    return float((np.abs(got - want) / np.abs(want)).max())


def check_against_reference(world, ref, f0, sp, fl, fs, fft, exact):
    """One call with a different ratio per utterance (and a scale from SCALES) against the restatement: f0 bit for bit,
    the envelope bit for bit where `exact` (host libm), else within 1e-12 relative.  Ratio 1.0 is compared like the
    others: the restatement takes the log / exp round trip there too, as the reference does.  Returns the worst
    envelope error."""
    ratios = ratios_for(fft)[:len(fl)]
    scales = [SCALES[u % len(SCALES)] for u in range(len(fl))]
    assert int(fft / 2.0 * ratios[-1]) == 1
    gf, gs = modify(world, f0, sp, fs, fft, scales, ratios, fl)
    worst = 0.0
    for u, L in enumerate(fl):
        wf, ws = ref_modify(ref, f0[u, :L], sp[u, :L], fs, fft, scales[u], ratios[u])
        assert np.array_equal(gf[u, :L], wf), f"utterance {u}: f0 differs"
        assert np.isfinite(ws).all() and (ws > 0).all()
        if exact:
            assert np.array_equal(gs[u, :L], ws), f"fs {fs} fft {fft} ratio {ratios[u]}: envelope differs " \
                f"(worst {rel_worst(gs[u, :L], ws):.2e} relative)"
        else:
            e = rel_worst(gs[u, :L], ws)
            assert e <= 1e-12, f"fs {fs} fft {fft} ratio {ratios[u]}: {e:.2e} relative"
            worst = max(worst, e)
    return worst


def check_golden(world, ref, golden, exact):
    """The fixture's envelope rows (CheapTrick of vaiueo2d, fft 1024 at 16 kHz), one utterance per ratio."""
    fs, fft = int(golden["fs"]), int(golden["fft_size"])
    sp = np.repeat(golden["sp"][None], 7, axis=0)
    f0 = np.repeat(golden["f0_stonemask"][None], 7, axis=0)
    L = sp.shape[1]
    fl = [L, L - 3, L - 10, L, L - 1, L - 40, L - 2]
    return check_against_reference(world, ref, f0, sp, fl, fs, fft, exact)


def check_analysed(world, ref, fs, fft, exact):
    f0, sp, fl = analysed_full_rows(world, fs, fft)
    assert (f0 > 0).sum() > 20
    return check_against_reference(world, ref, f0, sp, fl, fs, fft, exact)


def check_identity_and_bounds(world):
    """A NULL array leaves its rows bit-identical; frames beyond f0_lengths and a padded utterance keep their sentinel."""
    fs, fft, L, n = 16000, 512, 37, 4
    bins = fft // 2 + 1
    rng = np.random.default_rng(5)
    fl = [L, 20, 1, 33]
    f0 = np.full((n + 1, L), -3.0)
    sp = np.full((n + 1, L, bins), -5.0)
    for u in range(n):
        f0[u, :fl[u]] = np.where(rng.uniform(size=fl[u]) < 0.7, rng.uniform(80, 400, size=fl[u]), 0.0)
        sp[u, :fl[u]] = np.exp(rng.normal(size=(fl[u], bins)))
    scales, ratios = [1.5, 0.5, 2.0, 1.0], [0.7, 1.3, 2.0, 1.0]

    def run(sc, ra, with_f0=True, with_sp=True):
        F, S = pc.make(world, f0.copy()), pc.make(world, sp.copy())
        world._use_current_stream()
        rc = world.lib.world_b200_modify_batch(world._h, _ptr(F) if with_f0 else None, (C.c_int * n)(*fl), n, L,
                                               _ptr(S) if with_sp else None, fft, fs, _doubles(sc), _doubles(ra))
        world.synchronize()
        assert rc == 0, world.lib.world_b200_last_error(world._h)
        return pc.to_np(F), pc.to_np(S)

    gf, gs = run(scales, None, with_sp=False)
    assert np.array_equal(gs, sp) and not np.array_equal(gf, f0)
    gf2, gs2 = run(None, ratios, with_f0=False)
    assert np.array_equal(gf2, f0) and not np.array_equal(gs2, sp)
    gf3, gs3 = run(None, None, with_f0=False, with_sp=False)
    assert np.array_equal(gf3, f0) and np.array_equal(gs3, sp)
    gf, gs = run(scales, ratios)
    for u in range(n):
        assert (gf[u, fl[u]:] == -3.0).all() and (gs[u, fl[u]:] == -5.0).all(), f"utterance {u}: padding written"
        assert np.array_equal(gf[u, :fl[u]], f0[u, :fl[u]] * scales[u])
    assert (gf[n] == -3.0).all() and (gs[n] == -5.0).all(), "the padded utterance was written"


def _ptr(a):
    return cs._ptr(a)


def _doubles(v):
    return None if v is None else (C.c_double * len(v))(*v)


# ---- fused equals stepwise -------------------------------------------------------------------------------------------
def quantised(y):
    """wavwrite's 16-bit quantisation of a waveform: truncation toward zero, then the clamp."""
    return np.clip(np.trunc(y * 32767.0), -32768, 32767).astype(np.int16)


def stepwise(world, f0, csp, cap, fft, fp, fs, y_len, fl, yl, scales, ratios):
    """decode_spectral_envelope -> modify -> decode_aperiodicity -> synthesis of the same library."""
    dims = int(csp.shape[-1])
    f0 = f0.clone() if hasattr(f0, "clone") else f0.copy()
    sp = world.decode_spectral_envelope(csp, fs, fft, dims, f0_lengths=fl)
    if scales is not None or ratios is not None:
        world.modify(f0, sp, fs, fft, f0_scale=scales, spectral_ratio=ratios, f0_lengths=fl)
    ap = world.decode_aperiodicity(cap, fs, fft, f0_lengths=fl)
    y = world.synthesis(f0, sp, ap, fft, fp, fs, y_len, f0_lengths=fl, y_lengths=yl)
    world.synchronize()
    return pc.to_np(y)


def fused(world, f0, csp, cap, fft, fp, fs, y_len, fl, yl, scales, ratios, nbit=0):
    y = world.synthesis_coded(f0, csp, cap, fft, fp, fs, y_len, f0_lengths=fl, y_lengths=yl,
                              dtype="int16" if nbit == 16 else None, f0_scale=scales, spectral_ratio=ratios)
    world.synchronize()
    return pc.to_np(y)


def call_modified_raw(world, f0, csp, cap, fft, fp, fs, y_len, fl, yl, scales, ratios, nbit):
    """world_b200_synthesis_coded_batch_modified called directly, so NULL arrays reach the library as NULL."""
    n = int(f0.shape[0])
    y = pc.make(world, np.zeros((n, y_len)), dtype=np.int16 if nbit == 16 else np.float64)
    world._use_current_stream()
    rc = world.lib.world_b200_synthesis_coded_batch_modified(
        world._h, _ptr(f0), (C.c_int * n)(*fl), n, int(f0.shape[1]), _ptr(csp), int(csp.shape[-1]), _ptr(cap), fft, fp,
        fs, (C.c_int * n)(*yl), y_len, _doubles(scales), _doubles(ratios), nbit, _ptr(y))
    world.synchronize()
    assert rc == 0, world.lib.world_b200_last_error(world._h)
    return pc.to_np(y)


def check_fused_equals_stepwise(world, fs=16000, fp=5.0, dims=60):
    """A ragged batch with a different (scale, ratio) per utterance, nbit 0 and 16; NULL arrays give the unmodified
    calls; only-one-half calls equal their chains too."""
    f0, csp, cap, fl, lens = cs.analysed_rows(world, fs, fp, dims)
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    Y = max(yl)
    f0_in, csp_in = f0.copy(), csp.copy()
    F, S, A = pc.make(world, f0), pc.make(world, csp), pc.make(world, cap)
    scales, ratios = [1.5, 0.5, 2.0], [0.85, 1.3, 2.0 / fft]
    for sc, ra in ((scales, ratios), (scales, None), (None, ratios)):
        want = stepwise(world, F, S, A, fft, fp, fs, Y, fl, yl, sc, ra)
        got = fused(world, F, S, A, fft, fp, fs, Y, fl, yl, sc, ra)
        for u in range(len(fl)):
            assert np.abs(want[u, :yl[u]]).max() > 1e-4, f"utterance {u} is silent"
        assert np.array_equal(got, want), f"scales {sc} ratios {ra}: differs from the stepwise chain"
        got16 = fused(world, F, S, A, fft, fp, fs, Y, fl, yl, sc, ra, nbit=16)
        assert np.array_equal(got16, quantised(want)), f"scales {sc} ratios {ra}: pcm16 differs"
    assert np.array_equal(pc.to_np(F), f0_in) and np.array_equal(pc.to_np(S), csp_in), "the caller's rows were changed"
    plain = cs.coded(world, F, S, A, fft, fp, fs, Y, fl, yl)
    assert np.array_equal(call_modified_raw(world, F, S, A, fft, fp, fs, Y, fl, yl, None, None, 0), plain)
    plain16 = pc.to_np(world.synthesis_coded(F, S, A, fft, fp, fs, Y, f0_lengths=fl, y_lengths=yl, dtype="int16"))
    world.synchronize()
    assert np.array_equal(call_modified_raw(world, F, S, A, fft, fp, fs, Y, fl, yl, None, None, 16), plain16)


def check_small_budget(world):
    """At the smallest scratch budget the modified call runs in several passes and gives the one-pass result and the
    stepwise chain bit for bit."""
    fs, n_utt, secs, fft, dims = 16000, 5, 2.0, 1024, 40
    n = int(secs * fs)
    ylens = [n - 1337 * u for u in range(n_utt)]
    L = int(secs * 200) + 1
    flens = [L - 7 * u for u in range(n_utt)]
    scales, ratios = [1.2, 0.8, 1.0, 1.5, 0.6], [1.1, 0.9, 1.0, 1.3, 0.7]
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs, launches = [], []
        for w in (world, small):
            f0, csp, cap = cs.envelope_rows(w, np.random.default_rng(41), fs, fft, dims, flens, L)
            before = w.launch_count()
            outs.append(fused(w, f0, csp, cap, fft, 5.0, fs, n, flens, ylens, scales, ratios))
            launches.append(w.launch_count() - before)
        want = stepwise(world, *cs.envelope_rows(world, np.random.default_rng(41), fs, fft, dims, flens, L), fft, 5.0,
                        fs, n, flens, ylens, scales, ratios)
    finally:
        small.close()
    assert launches[1] >= 2 * launches[0], f"launches: {launches[0]} in one pass, {launches[1]} at the small budget"
    assert np.array_equal(outs[0], outs[1]), "chunked result differs"
    assert np.array_equal(outs[0], want), "differs from the stepwise chain"


def check_scaled_high_f0(world):
    """Scale 3.0 on a 500 Hz contour: 1,500 pulses per second, beyond the 1,200 the arrays are first laid out for, so
    the pass is laid out again from the counts of the scaled copy (one more time-base and one more f0 copy launch than
    the same call at scale 1.0); the result equals the stepwise chain."""
    fs, fft, dims, secs = 16000, 1024, 40, 1.0
    n = int(secs * fs)
    L = int(secs * 200) + 1
    flens, ylens = [L, L - 11, L - 23], [n, n - 901, n - 1802]
    f0, csp, cap = cs.envelope_rows(world, np.random.default_rng(43), fs, fft, dims, flens, L, f0_hz={1: 500.0})
    scales, ratios = [1.0, 3.0, 1.0], [1.0, 1.25, 0.9]
    want = stepwise(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens, scales, ratios)
    before = world.launch_count()
    got = fused(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens, scales, ratios)
    relaid = world.launch_count() - before
    before = world.launch_count()
    fused(world, f0, csp, cap, fft, 5.0, fs, n, flens, ylens, [1.0, 1.0, 1.0], ratios)
    assert relaid == world.launch_count() - before + 2, "the scaled 1.5 kHz utterance did not take the relaid pass"
    assert np.array_equal(got, want), "scaled above 1.2 kHz: differs from the stepwise chain"


def check_host_equals_device(world, pinned=False, fs=16000, fp=5.0, dims=60):
    """synthesis_coded_host with the factors equals the device call, nbit 0 and 16 (chunked at the small budget)."""
    f0, csp, cap, fl, lens = cs.analysed_rows(world, fs, fp, dims, seeds=(421, 422, 423))
    fft = world.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    Y = max(yl)
    scales, ratios = [0.7, 1.5, 1.0], [1.2, 0.8, 1.0]
    F, S, A = pc.make(world, f0), pc.make(world, csp), pc.make(world, cap)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        for nbit in (0, 16):
            want = fused(world, F, S, A, fft, fp, fs, Y, fl, yl, scales, ratios, nbit=nbit)
            hosts = [f0, csp, cap]
            out = None
            if pinned:
                import torch
                hosts = [torch.from_numpy(a).pin_memory() for a in hosts]
                out = torch.zeros((len(fl), Y), dtype=torch.int16 if nbit == 16 else torch.float64).pin_memory()
            for w in (world, small):
                got = w.synthesis_coded_host(*hosts, fft, fp, fs, Y, nbit=nbit, f0_lengths=fl, y_lengths=yl, out=out,
                                             f0_scale=scales, spectral_ratio=ratios)
                assert np.array_equal(np.asarray(got), want), f"nbit {nbit}: the host call differs from the device call"
    finally:
        small.close()


# ---- invalid input -------------------------------------------------------------------------------------------------
def check_invalid(world):
    """Every bad factor or argument is EINVAL before any work: nothing is launched, the outputs keep their sentinels,
    and last_error names the first bad utterance."""
    fs, fp, fft, dims, L, n, Y = 16000, 5.0, 1024, 40, 41, 5, 3200
    bins = fft // 2 + 1
    rng = np.random.default_rng(47)
    fl, yl = [L, L - 5, L - 9, L, L - 2], [Y, Y - 100, Y - 333, Y, Y - 7]
    f0c, csp, cap = cs.envelope_rows(world, rng, fs, fft, dims, fl, L)
    f0 = pc.make(world, np.full((n, L), 150.0))
    sp = pc.make(world, np.full((n, L, bins), 0.25))
    y = pc.make(world, np.full((n, Y), -7.0))
    lib = world.lib
    good_s, good_r = [1.0] * n, [1.0] * n
    tiny = float(np.nextafter(2.0 / fft, 0.0))   # (int)(fft / 2.0 * tiny) == 0

    def bad(vals, u, v):
        vals = list(vals)
        vals[u] = v
        vals[4] = v
        return vals

    def err():
        return lib.world_b200_last_error(world._h).decode()

    def run(fn):
        world._use_current_stream()
        before = world.launch_count()
        rc = fn()
        world.synchronize()
        return rc, world.launch_count() - before

    def modify(sc=good_s, ra=good_r, fft_size=fft, f=True, s=True, lens=fl):
        return lambda: lib.world_b200_modify_batch(world._h, _ptr(f0) if f else None, (C.c_int * n)(*lens), n, L,
                                                   _ptr(sp) if s else None, fft_size, fs, _doubles(sc), _doubles(ra))

    def synth(sc=good_s, ra=good_r, nbit=0):
        return lambda: lib.world_b200_synthesis_coded_batch_modified(
            world._h, _ptr(f0c), (C.c_int * n)(*fl), n, L, _ptr(csp), dims, _ptr(cap), fft, fp, fs, (C.c_int * n)(*yl),
            Y, _doubles(sc), _doubles(ra), nbit, _ptr(y))

    cases = []
    for what, v in (("0", 0.0), ("-1", -1.0), ("NaN", float("nan")), ("inf", float("inf")), ("-0", -0.0)):
        cases.append((f"modify: spectral_ratio {what}", modify(ra=bad(good_r, 2, v)), "spectral_ratio[2]"))
        cases.append((f"modify: f0_scale {what}", modify(sc=bad(good_s, 1, v)), "f0_scale[1]"))
        cases.append((f"synthesis: spectral_ratio {what}", synth(ra=bad(good_r, 3, v)), "spectral_ratio[3]"))
        cases.append((f"synthesis: f0_scale {what}", synth(sc=bad(good_s, 0, v)), "f0_scale[0]"))
    cases += [
        ("modify: c == 0", modify(ra=bad(good_r, 2, tiny)), "spectral_ratio[2]"),
        ("synthesis: c == 0", synth(ra=bad(good_r, 1, tiny)), "spectral_ratio[1]"),
        ("modify: fft_size 1000", modify(fft_size=1000), "fft_size"),
        ("modify: fft_size 8192", modify(fft_size=8192), "fft_size"),
        ("modify: f0 NULL with f0_scale", modify(f=False), "f0_scale"),
        ("modify: spectrogram NULL with spectral_ratio", modify(s=False), "spectral_ratio"),
        ("modify: f0 length beyond its row", modify(lens=[L, L, L + 1, L, L]), "f0_lengths[2]"),
        ("synthesis: nbit 8", synth(nbit=8), "nbit"),
    ]
    for what, fn, named in cases:
        rc, launched = run(fn)
        assert rc == EINVAL, f"{what}: returned {rc}"
        assert launched == 0, f"{what}: {launched} kernels launched"
        assert named in err(), f"{what}: last_error {err()!r} does not name {named}"
        assert (pc.to_np(f0) == 150.0).all() and (pc.to_np(sp) == 0.25).all() and (pc.to_np(y) == -7.0).all(), \
            f"{what}: an output was written"
    # the host call checks the same before it queues anything
    yh = np.full((n, Y), -7.0)
    rc = lib.world_b200_synthesis_coded_host_modified(
        world._h, pc.to_np(f0c).ctypes.data, (C.c_int * n)(*fl), n, L, np.ascontiguousarray(pc.to_np(csp)).ctypes.data,
        dims, np.ascontiguousarray(pc.to_np(cap)).ctypes.data, fft, fp, fs, (C.c_int * n)(*yl), Y, _doubles(good_s),
        _doubles(bad(good_r, 2, -2.0)), 0, yh.ctypes.data)
    assert rc == EINVAL and "spectral_ratio[2]" in err() and (yh == -7.0).all()
    # the smallest ratio with c == 1 is accepted; the context keeps working
    rc, launched = run(modify(ra=bad(good_r, 2, 2.0 / fft)))
    assert rc == 0 and launched > 0
    rc, launched = run(synth(sc=[1.2] * n, ra=[0.9] * n))
    assert rc == 0 and launched > 0


# ---- the reference's own demo ---------------------------------------------------------------------------------------
def write_fixture_wav(golden, path):
    import wave
    with wave.open(path, "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(int(golden["fs"]))
        w.writeframes(np.ascontiguousarray(golden["pcm"]).astype("<i2").tobytes())


def read_wav16(path):
    import wave
    with wave.open(path, "rb") as w:
        assert w.getsampwidth() == 2 and w.getnchannels() == 1
        return np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").astype(np.int64)


def run_ref_demo(golden, d, shift, ratio):
    """test/test.cpp compiled unchanged: in.wav -> 01out.wav (Synthesis of the modified parameters, 16 bit)."""
    write_fixture_wav(golden, os.path.join(d, "in.wav"))
    r = subprocess.run([REF_DEMO, "in.wav", "out.wav", repr(shift), repr(ratio)], cwd=d, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return read_wav16(os.path.join(d, "01out.wav"))


def library_demo_chain(world, golden, shift, ratio):
    """The demo's chain on the library: Harvest (floor 40), CheapTrick (floor 71), D4C (threshold 0.85), modify,
    Synthesis, then wavwrite's quantisation."""
    fs = int(golden["fs"])
    x = (golden["pcm"].astype(np.float64) / 32768.0)[None]
    X = pc.make(world, x)
    ho = world.harvest_option()
    ho.f0_floor, ho.frame_period = 40.0, 5.0
    t, f0, fl = world.harvest(X, fs, ho)
    co = world.cheaptrick_option(fs)
    assert co.f0_floor == 71.0
    sp = world.cheaptrick(X, fs, t, f0, co)
    do = world.d4c_option()
    do.threshold = 0.85
    ap = world.d4c(X, fs, t, f0, co.fft_size, do)
    world.modify(f0, sp, fs, co.fft_size, f0_scale=shift, spectral_ratio=ratio)
    L = fl[0]
    y_len = int((L - 1) * 5.0 / 1000.0 * fs) + 1
    y = world.synthesis(f0, sp, ap, co.fft_size, 5.0, fs, y_len)
    world.synchronize()
    return quantised(pc.to_np(y)[0]).astype(np.int64)


def check_ref_demo(world, golden, d):
    for shift, ratio in ((1.5, 0.85), (0.7, 1.3)):
        want = run_ref_demo(golden, d, shift, ratio)
        got = library_demo_chain(world, golden, shift, ratio)
        assert got.shape == want.shape
        assert np.abs(want).max() > 1000
        diff = int(np.abs(got - want).max())
        assert diff <= 1, f"shift {shift} ratio {ratio}: {diff} LSB from the reference demo"
