"""Checks of pitch and formant curves (world_b200_modify_curves, world_b200_modify_curves_packed,
world_b200_transform_packed_curves and world_b200_transform_host_packed_curves): one f0 factor and one spectral ratio
per frame.  The same assertions run against the host emulation (CPU) and the CUDA library (-m gpu).

The oracles: the per-utterance factor calls (constant curves must give their result bit for bit), the factor call on
the same rows laid out as one-frame utterances (each frame is its own ParameterModification), the reference's own
interp1 frame by frame (modify_common.ref_modify), and for the transformation the stepwise chain analyze_packed ->
modify_curves_packed -> synthesis_packed."""
import ctypes as C
import os

import numpy as np

import modify_common as mc
import packed_synthesis_common as ps
import test_parity_common as pc
import transform_packed_common as tpc

EINVAL = 3
SIZES = (16, 32, 64, 128, 256, 512, 1024, 2048, 4096)
SENTINEL = -5.0


def _doubles(world, a):
    return pc.make(world, np.ascontiguousarray(a, dtype=np.float64))


def err(world):
    return world.lib.world_b200_last_error(world._h).decode()


# ---- rows --------------------------------------------------------------------------------------------------------
def constant_case(rng, frames=(3, 1, 0, 2)):
    """One utterance per (fft_size, ratio) of SIZES x modify_common.ratios_for, with frame counts cycling through
    `frames` (0: an empty utterance), a scale per utterance, and envelope rows exp(normal) in rows wider than every size
    whose other entries hold SENTINEL."""
    sizes, ratios = [], []
    for fft in SIZES:
        for r in mc.ratios_for(fft):
            sizes.append(fft)
            ratios.append(r)
    n = len(sizes)
    lens = [frames[u % len(frames)] for u in range(n)]
    scales = [mc.SCALES[u % len(mc.SCALES)] for u in range(n)]
    return sizes, ratios, scales, lens


def padded_rows(rng, sizes, lens, width, L):
    n = len(sizes)
    f0 = np.full((n, L), SENTINEL)
    sp = np.full((n, L, width), SENTINEL)
    for u in range(n):
        b = sizes[u] // 2 + 1
        f0[u, :lens[u]] = rng.uniform(80.0, 400.0, lens[u])
        sp[u, :lens[u], :b] = np.exp(rng.normal(size=(lens[u], b)))
    return f0, sp


def pack(f0, sp, lens):
    fo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return (np.concatenate([f0[u, :m] for u, m in enumerate(lens)]),
            np.concatenate([sp[u, :m] for u, m in enumerate(lens)]), fo)


def guarded_rows(world, f0, sp):
    """Device rows with ps.GUARD sentinel frames on either side: (guarded f0, f0 view, guarded sp, sp view)."""
    gf, f = ps.guarded(world, f0, SENTINEL)
    gs, s = ps.guarded(world, sp, SENTINEL)
    return gf, f, gs, s


# ---- 1. constant curves equal the factor calls -------------------------------------------------------------------
def check_constant_equals_factors(world):
    """curve[f] = factor[u] on every frame of utterance u: modify_curves equals modify (per-utterance sizes) and
    modify_curves_packed equals modify_packed, bit for bit, at every size from 16 to 4096 and the ratios 0.5, 0.83,
    1.0, 1.2, 2.0, 3.7 and 2 / fft; frames past each length, bins past each size and guard frames keep their
    sentinels; an empty utterance is allowed."""
    rng = np.random.default_rng(71)
    sizes, ratios, scales, lens = constant_case(rng)
    n, L, width = len(sizes), 4, max(SIZES) // 2 + 3
    f0, sp = padded_rows(rng, sizes, lens, width, L)
    fc = np.full((n, L), np.nan)   # past each length the curve is not read
    rc = np.full((n, L), np.nan)
    for u in range(n):
        fc[u, :lens[u]], rc[u, :lens[u]] = scales[u], ratios[u]
    F1, S1 = pc.make(world, f0.copy()), pc.make(world, sp.copy())
    world.modify(F1, S1, 16000, sizes, f0_scale=scales, spectral_ratio=ratios, f0_lengths=lens)
    F2, S2 = pc.make(world, f0.copy()), pc.make(world, sp.copy())
    world.modify_curves(F2, S2, 16000, sizes, f0_curve=_doubles(world, fc), spectral_ratio_curve=_doubles(world, rc),
                        f0_lengths=lens)
    world.synchronize()
    want_f, want_s = pc.to_np(F1), pc.to_np(S1)
    got_f, got_s = pc.to_np(F2), pc.to_np(S2)
    assert np.array_equal(got_f, want_f), "padded: f0 differs from modify"
    for u in range(n):
        assert np.array_equal(got_s[u], want_s[u]), f"padded: fft {sizes[u]} ratio {ratios[u]}: envelope differs"
        b = sizes[u] // 2 + 1
        assert (got_s[u, :, b:] == SENTINEL).all() and (got_s[u, lens[u]:] == SENTINEL).all(), \
            f"padded utterance {u}: a sentinel was written"
        assert (got_f[u, lens[u]:] == SENTINEL).all()
    # packed, between guard frames
    pf0, psp, fo = pack(f0, sp, lens)
    pfc = np.concatenate([fc[u, :m] for u, m in enumerate(lens)])
    prc = np.concatenate([rc[u, :m] for u, m in enumerate(lens)])
    gf1, F1, gs1, S1 = guarded_rows(world, pf0, psp)
    world.modify_packed(F1, S1, fo, 16000, fft_size=sizes, f0_scale=scales, spectral_ratio=ratios)
    gf2, F2, gs2, S2 = guarded_rows(world, pf0, psp)
    world.modify_curves_packed(F2, S2, fo, 16000, fft_size=sizes, f0_curve=_doubles(world, pfc),
                               spectral_ratio_curve=_doubles(world, prc))
    world.synchronize()
    assert np.array_equal(pc.to_np(gf2), pc.to_np(gf1)), "packed: f0 differs from modify_packed"
    assert np.array_equal(pc.to_np(gs2), pc.to_np(gs1)), "packed: envelope differs from modify_packed"
    assert ps.untouched(gf2, SENTINEL) and ps.untouched(gs2, SENTINEL), "packed: a guard frame was written"
    got = pc.to_np(S2)
    for u in range(n):
        assert (got[fo[u]:fo[u + 1], sizes[u] // 2 + 1:] == SENTINEL).all(), f"packed utterance {u}: bins written"


# ---- 2. and 3. each frame is its own ParameterModification -------------------------------------------------------
def real_rows(world, golden, frames=48):
    """Envelope and f0 rows of real speech at mixed sizes, packed: the fixture's CheapTrick rows (fft 1024, 16 kHz) and
    the library's own analysis at fft 512 and 2048 (16 kHz), a few utterances of each.  Returns (f0 [F], sp [F, W],
    f_offsets, sizes) on the host, fs 16000."""
    parts = []
    g_sp, g_f0 = golden["sp"], golden["f0_stonemask"]
    for k in range(2):   # two stretches of the fixture
        a = 60 + 90 * k
        parts.append((1024, g_f0[a:a + frames], g_sp[a:a + frames]))
    for fft in (512, 2048):
        f0, sp, fl = mc.analysed_full_rows(world, 16000, fft)
        for u in range(2):
            m = min(fl[u], frames)
            parts.append((fft, f0[u, :m], sp[u, :m]))
    width = max(p[0] for p in parts) // 2 + 1
    sizes = [p[0] for p in parts]
    lens = [len(p[1]) for p in parts]
    fo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    F = int(fo[-1])
    f0 = np.zeros(F)
    sp = np.full((F, width), SENTINEL)
    for u, (fft, a, b) in enumerate(parts):
        f0[fo[u]:fo[u + 1]] = a
        sp[fo[u]:fo[u + 1], :fft // 2 + 1] = b
    return f0, sp, fo, sizes


def varying_curves(rng, fo, sizes):
    """Per-frame curves: ratios mixing smooth random values with the node-hitting 0.5, 1.0 and 2.0 and the smallest
    ratio 2 / fft; factors a smooth random curve."""
    F = int(fo[-1])
    rc, fc = np.empty(F), np.empty(F)
    for u, fft in enumerate(sizes):
        m = int(fo[u + 1] - fo[u])
        t = np.arange(m)
        smooth = np.exp(0.5 * np.sin(2 * np.pi * t / max(m, 1) * rng.uniform(0.5, 2.0) + rng.uniform(0, 6.3)))
        pool = np.array([0.5, 1.0, 2.0, 2.0 / fft, 3.7, 0.83])
        pick = rng.uniform(size=m) < 0.35
        r = np.where(pick, pool[rng.integers(0, len(pool), m)], smooth)
        rc[fo[u]:fo[u + 1]] = r
        fc[fo[u]:fo[u + 1]] = np.exp(0.4 * np.sin(2 * np.pi * t / 40.0 + u))
    return fc, rc


def curves_packed(world, f0, sp, fo, sizes, fc, rc, fs=16000):
    F, S = pc.make(world, f0.copy()), pc.make(world, sp.copy())
    world.modify_curves_packed(F, S, fo, fs, fft_size=sizes, f0_curve=None if fc is None else _doubles(world, fc),
                               spectral_ratio_curve=None if rc is None else _doubles(world, rc))
    world.synchronize()
    return pc.to_np(F), pc.to_np(S)


def check_frames_equal_lone_calls(world, golden):
    """modify_curves_packed on real utterances equals modify_packed on the same rows laid out as one-frame utterances
    (f_offsets 0..F, fft_sizes[f] the frame's utterance's, factors the curves), bit for bit."""
    f0, sp, fo, sizes = real_rows(world, golden)
    fc, rc = varying_curves(np.random.default_rng(73), fo, sizes)
    gf, gs = curves_packed(world, f0, sp, fo, sizes, fc, rc)
    F = int(fo[-1])
    frame_sizes = [sizes[u] for u in range(len(sizes)) for _ in range(int(fo[u + 1] - fo[u]))]
    Fw, Sw = pc.make(world, f0.copy()), pc.make(world, sp.copy())
    world.modify_packed(Fw, Sw, np.arange(F + 1, dtype=np.int64), 16000, fft_size=frame_sizes, f0_scale=fc,
                        spectral_ratio=rc)
    world.synchronize()
    assert np.array_equal(gf, pc.to_np(Fw)), "f0 differs from the one-frame calls"
    want = pc.to_np(Sw)
    for f in range(F):
        assert np.array_equal(gs[f], want[f]), f"frame {f} (fft {frame_sizes[f]}, ratio {rc[f]!r}) differs"


def check_vs_reference(world, ref, golden, exact):
    """Each frame against the reference's ParameterModification of that one frame (its own interp1): bit for bit where
    `exact` (the emulation's host libm), else within 1e-12 relative; f0 bit for bit.  Returns the worst error."""
    f0, sp, fo, sizes = real_rows(world, golden, frames=24)
    fc, rc = varying_curves(np.random.default_rng(79), fo, sizes)
    gf, gs = curves_packed(world, f0, sp, fo, sizes, fc, rc)
    worst = 0.0
    for u, fft in enumerate(sizes):
        b = fft // 2 + 1
        for f in range(int(fo[u]), int(fo[u + 1])):
            wf, ws = mc.ref_modify(ref, f0[f:f + 1], sp[f:f + 1, :b], 16000, fft, fc[f], rc[f])
            assert gf[f] == wf[0], f"frame {f}: f0 differs"
            what = f"frame {f} (fft {fft}, ratio {rc[f]!r})"
            if exact:
                assert np.array_equal(gs[f, :b], ws[0]), f"{what}: differs from the reference"
            else:
                e = mc.rel_worst(gs[f, :b], ws[0])
                assert e <= 1e-12, f"{what}: {e:.2e} relative"
                worst = max(worst, e)
            assert (gs[f, b:] == SENTINEL).all()
    return worst


def check_null_halves(world):
    """A NULL curve leaves its half bit-identical; n_utts 0 returns 0."""
    rng = np.random.default_rng(83)
    sizes, lens = [512, 64, 1024], [5, 0, 4]
    f0, sp = padded_rows(rng, sizes, lens, 513, 5)
    pf0, psp, fo = pack(f0, sp, lens)
    fc, rc = varying_curves(rng, fo, sizes)
    gf, gs = curves_packed(world, pf0, psp, fo, sizes, fc, None)
    assert np.array_equal(gs, psp) and not np.array_equal(gf, pf0)
    gf, gs = curves_packed(world, pf0, psp, fo, sizes, None, rc)
    assert np.array_equal(gf, pf0) and not np.array_equal(gs, psp)
    gf, gs = curves_packed(world, pf0, psp, fo, sizes, None, None)
    assert np.array_equal(gf, pf0) and np.array_equal(gs, psp)
    lib = world.lib
    assert lib.world_b200_modify_curves_packed(world._h, None, 0, None, None, 0, None, 16000, None, None) == 0
    assert lib.world_b200_modify_curves(world._h, None, None, 0, 0, None, 0, None, 16000, None, None) == 0


# ---- 4. the transformation ---------------------------------------------------------------------------------------
def transform_case(world, n_utts=4, seed=41):
    K = tpc.Case(world, 16000, 3200, n_utts, family="none", seed=seed)
    fo = world.packed_frames(K.fs, K.xo, K.fp)
    return K, fo


def transform_curves(world, K, fc, rc, nbit_out, host=False, nbit=0):
    data, _ = K.P.x_packed(nbit)
    dtype = "int16" if nbit_out == 16 else None
    if host:
        y, yo = world.transform_host_packed_curves(data, nbit, K.xo, K.fs, K.c.ao, f0_curve=fc, spectral_ratio_curve=rc,
                                                   time_scale=K.tscales, dtype=dtype, **K.c.kw)
    else:
        y, yo = world.transform_packed_curves(pc.make(world, data, data.dtype), nbit, K.xo, K.fs, K.c.ao,
                                              f0_curve=None if fc is None else _doubles(world, fc),
                                              spectral_ratio_curve=None if rc is None else _doubles(world, rc),
                                              time_scale=K.tscales, dtype=dtype, **K.c.kw)
    world.synchronize()
    return pc.to_np(y), yo


def stepwise(world, K, fc, rc):
    """analyze_packed -> modify_curves_packed -> synthesis_packed of each utterance at frame_period * time_scale[u]."""
    data, _ = K.P.x_packed(0)
    t, f0, sp, ap, fo = world.analyze_packed(pc.make(world, data), K.xo, K.fs, K.c.ao, **K.c.kw)
    world.modify_curves_packed(f0, sp, fo, K.fs, fft_size=K.c.sizes, f0_curve=_doubles(world, fc),
                               spectral_ratio_curve=_doubles(world, rc))
    world.synchronize()
    f0, sp, ap = pc.to_np(f0), pc.to_np(sp), pc.to_np(ap)
    out = []
    for u in range(K.n):
        a, b = int(fo[u]), int(fo[u + 1])
        fp = K.fp * K.tscales[u]
        Y = world.transform_samples(K.fs, int(K.xo[u + 1] - K.xo[u]), K.fp, K.tscales[u])
        y = world.synthesis_packed(pc.make(world, f0[a:b].copy()), pc.make(world, sp[a:b].copy()),
                                   pc.make(world, ap[a:b].copy()), [0, b - a], [K.c.sizes[u]], fp, K.fs, [0, Y])
        world.synchronize()
        out.append(pc.to_np(y))
    return out


def check_transform_equals_stepwise(world):
    """Varying curves: transform_packed_curves equals the stepwise chain bit for bit, float64 out and int16 out (the
    pcm16 rule of the stepwise samples); the host call equals the device call, at the default chunks and one
    utterance per chunk (curve frames read from each chunk's own copy)."""
    K, fo = transform_case(world)
    fc, rc = varying_curves(np.random.default_rng(89), fo, K.c.sizes)
    want = stepwise(world, K, fc, rc)
    got, yo = transform_curves(world, K, fc, rc, 0)
    got16, yo16 = transform_curves(world, K, fc, rc, 16)
    assert np.array_equal(yo, yo16)
    for u in range(K.n):
        seg = got[yo[u]:yo[u + 1]]
        assert len(seg) == len(want[u]) and np.abs(want[u]).max() > 1e-4
        assert np.array_equal(seg, want[u]), f"utterance {u}: differs from the stepwise chain"
        assert np.array_equal(got16[yo[u]:yo[u + 1]], mc.quantised(want[u])), f"utterance {u}: int16 differs"
    old = os.environ.get("WB_HOST_CHUNK")
    try:
        for chunk in (None, "1"):
            if chunk:
                os.environ["WB_HOST_CHUNK"] = chunk
            else:
                os.environ.pop("WB_HOST_CHUNK", None)
            for nbit_out, dev in ((0, got), (16, got16)):
                h, ho = transform_curves(world, K, fc, rc, nbit_out, host=True)
                assert np.array_equal(ho, yo) and np.array_equal(h, dev), f"chunk {chunk}, nbit_out {nbit_out}: host differs"
    finally:
        if old is None:
            os.environ.pop("WB_HOST_CHUNK", None)
        else:
            os.environ["WB_HOST_CHUNK"] = old


def check_transform_constant_equals_factors(world):
    """Constant curves: transform_packed_curves and transform_host_packed_curves equal transform_packed with those
    factors, float64 and int16 out, from int16 input too; f0 curve only equals f0_scale only."""
    K, fo = transform_case(world, n_utts=5, seed=43)
    scale, ratio = tpc.factors(K.n, "both")
    fc = np.concatenate([[scale[u]] * int(fo[u + 1] - fo[u]) for u in range(K.n)])
    rc = np.concatenate([[ratio[u]] * int(fo[u + 1] - fo[u]) for u in range(K.n)])
    for nbit, nbit_out, with_ratio in ((0, 0, True), (16, 16, True), (16, 0, False)):
        data, _ = K.P.x_packed(nbit)
        want, wo = world.transform_packed(pc.make(world, data, data.dtype), nbit, K.xo, K.fs, K.c.ao, f0_scale=scale,
                                          spectral_ratio=ratio if with_ratio else None, time_scale=K.tscales,
                                          dtype="int16" if nbit_out == 16 else None, **K.c.kw)
        world.synchronize()
        want = pc.to_np(want)
        r = rc if with_ratio else None
        for host in (False, True):
            got, go = transform_curves(world, K, fc, r, nbit_out, host=host, nbit=nbit)
            what = f"nbit {nbit} -> {nbit_out}, ratio curve {with_ratio}, host {host}"
            assert np.array_equal(go, wo) and np.array_equal(got, want), f"{what}: differs from transform_packed"


# ---- 5. invalid input --------------------------------------------------------------------------------------------
def check_invalid(world):
    """Bad curve values and bad offsets are EINVAL before anything is modified, naming the curve, utterance and frame;
    the rows and outputs keep their values.  Values past an utterance's frames are not read."""
    rng = np.random.default_rng(97)
    sizes, lens = [512, 1024, 256, 2048], [6, 4, 0, 5]
    f0, sp = padded_rows(rng, sizes, lens, 1025, 6)
    pf0, psp, fo = pack(f0, sp, lens)
    F = int(fo[-1])
    lib = world.lib
    good = np.ones(F)

    def packed(fc=good, rc=good, offs=fo):
        Fd, Sd = pc.make(world, pf0.copy()), pc.make(world, psp.copy())
        Fc, Rc = _doubles(world, fc), _doubles(world, rc)   # held until the call has returned
        world._use_current_stream()
        o = (C.c_longlong * len(offs))(*[int(v) for v in offs])
        rc_ = lib.world_b200_modify_curves_packed(world._h, mc._ptr(Fd), len(sizes), o, mc._ptr(Sd), 1025,
                                                  (C.c_int * 4)(*sizes), 16000, mc._ptr(Fc), mc._ptr(Rc))
        world.synchronize()
        return rc_, pc.to_np(Fd), pc.to_np(Sd)

    def at(u, f, v):
        c = good.copy()
        c[fo[u] + f] = v
        return c

    tiny = float(np.nextafter(2.0 / 1024, 0.0))
    cases = []
    for name, v in (("0", 0.0), ("-1", -1.0), ("NaN", float("nan")), ("inf", float("inf"))):
        cases.append((f"f0 {name}", dict(fc=at(3, 2, v)), "f0_curve", "utterance 3, frame 2"))
        cases.append((f"ratio {name}", dict(rc=at(1, 3, v)), "spectral_ratio_curve", "utterance 1, frame 3"))
    cases.append(("ratio below 2 / fft", dict(rc=at(1, 0, tiny)), "spectral_ratio_curve", "utterance 1, frame 0"))
    bad_off = fo.copy()
    bad_off[1], bad_off[2] = bad_off[2], bad_off[1]
    cases.append(("offsets", dict(offs=bad_off), "f_offsets", "utterance"))
    for what, kw, named, where in cases:
        rc_, gf, gs = packed(**kw)
        assert rc_ == EINVAL, f"{what}: returned {rc_}"
        assert named in err(world) and where in err(world), f"{what}: last_error {err(world)!r}"
        assert np.array_equal(gf, pf0) and np.array_equal(gs, psp), f"{what}: the rows were written"
    # 2 / 1024 itself keeps one bin; the first bad frame is named when there are several
    rc_, _, _ = packed(rc=at(1, 0, 2.0 / 1024))
    assert rc_ == 0, err(world)
    two = at(3, 4, 0.0)
    two[fo[0] + 1] = -2.0
    rc_, _, _ = packed(fc=two)
    assert rc_ == EINVAL and "utterance 0, frame 1" in err(world), err(world)
    # padded rows: NaN past each length is not read; a bad value inside one is named
    fcp = np.full(f0.shape, np.nan)
    for u in range(len(sizes)):
        fcp[u, :lens[u]] = 1.25
    Fd, Sd = pc.make(world, f0.copy()), pc.make(world, sp.copy())
    world.modify_curves(Fd, Sd, 16000, sizes, f0_curve=_doubles(world, fcp), f0_lengths=lens)
    world.synchronize()
    assert np.array_equal(pc.to_np(Fd)[0, :6], f0[0, :6] * 1.25)
    fcp[1, 3] = np.inf
    Fd, Fc = pc.make(world, f0.copy()), _doubles(world, fcp)
    world._use_current_stream()
    rc_ = lib.world_b200_modify_curves(world._h, mc._ptr(Fd), (C.c_int * 4)(*lens), 4, 6, None, 0,
                                       (C.c_int * 4)(*sizes), 16000, mc._ptr(Fc), None)
    world.synchronize()
    assert rc_ == EINVAL and "f0_curve[9]" in err(world) and "utterance 1, frame 3" in err(world), err(world)
    assert np.array_equal(pc.to_np(Fd), f0)


def check_transform_invalid(world):
    """A bad curve frame of the transformation is EINVAL before any work, naming its utterance and frame; y is
    untouched (device), and the host call rejects it the same way."""
    K, fo = transform_case(world, n_utts=3, seed=47)
    F = int(fo[-1])
    data, _ = K.P.x_packed(0)
    Y = int(world.transform_packed_samples(K.fs, K.xo, K.fp, K.tscales)[-1])
    for name, u, f, fcv, rcv in (("f0 0", 2, 5, 0.0, 1.0), ("ratio NaN", 1, 0, 1.0, np.nan)):
        fc, rc = np.ones(F), np.ones(F)
        (fc if name.startswith("f0") else rc)[fo[u] + f] = fcv if name.startswith("f0") else rcv
        yg, y = ps.guarded(world, np.zeros(Y), 7.0)
        before = pc.to_np(yg).copy()
        try:
            world.transform_packed_curves(pc.make(world, data), 0, K.xo, K.fs, K.c.ao, f0_curve=_doubles(world, fc),
                                          spectral_ratio_curve=_doubles(world, rc), time_scale=K.tscales, y=y, **K.c.kw)
            raise AssertionError(f"{name}: accepted")
        except AssertionError:
            raise
        except Exception as e:   # WorldError
            assert f"utterance {u}, frame {f}" in str(e), str(e)
        world.synchronize()
        assert np.array_equal(pc.to_np(yg), before), f"{name}: y was written"
        out = np.full(Y, 7.0)
        try:
            world.transform_host_packed_curves(data, 0, K.xo, K.fs, K.c.ao, f0_curve=fc, spectral_ratio_curve=rc,
                                               time_scale=K.tscales, out=out, **K.c.kw)
            raise AssertionError(f"{name}: the host call accepted it")
        except AssertionError:
            raise
        except Exception as e:
            assert f"utterance {u}, frame {f}" in str(e), str(e)
        assert (out == 7.0).all(), f"{name}: the host call wrote y"
