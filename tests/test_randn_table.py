"""The randn() stream table of a context.  Every utterance of every CheapTrick, D4C and Synthesis call consumes the
same stream from draw 0 (the reference reseeds randn() at each call), so a context keeps one table of it (wb_rng.cu,
rng_table_reserve) and a frame reads its draws at its stream offset there.  The table grows to the largest bound a call
asks for and only world_b200_trim() gives it back, so a call may find a table sized by a larger call, by a smaller one
it has to grow, or none.  Whatever the table's history, the rows must equal a fresh context's bit for bit:
  (a) CheapTrick + D4C on short utterances, then on longer ones at a larger fft_size (the table grows), then on the
      short ones again; against fresh contexts and the reference;
  (b) the same after trim();
  (c) analyze_batch in two lanes (sibling contexts, one table each) against one lane;
  (d) per-utterance CheapTrick / D4C options and packed analysis rows: each utterance equals its own one-option or
      padded call;
  (e) packed Synthesis and the packed voice transformation equal their padded forms.
Each check runs on the host emulation (CPU suite) and on the CUDA library (-m gpu)."""
import numpy as np
import pytest

import packed_common as pk
import packed_synthesis_common as ps
import spectral_options_common as so
import transform_packed_common as tp
from coded_batch_common import lane_slices
from test_parity_common import assert_close, make, to_np
from test_stage_paths import _contours

FS = 16000


def _fresh(world):
    from world_b200.api import World
    return World(device=world.device, lib_path=world.lib._name, array_module=world.xp)


def _batch(seed, n_utt, frames, fft):
    """n_utt utterances of `frames` 1 ms frames (ragged by 37 frames), their waveform long enough for every frame"""
    from synth import synth_batch
    fl = [frames - 37 * u for u in range(n_utt)]
    n = int(frames * FS / 1000) + FS // 50
    lens = [int(f * FS / 1000) + FS // 50 for f in fl]
    x = synth_batch(range(seed, seed + n_utt), FS, n).numpy()
    t, f = _contours(np.random.default_rng(seed), fl, frames)
    return x, t, f, lens, fl, fft


def _spectral(w, batch):
    x, t, f, lens, fl, fft = batch
    o = w.cheaptrick_option(FS)
    o.fft_size = fft
    xb, tb, fb = make(w, x), make(w, t), make(w, f)
    sp = w.cheaptrick(xb, FS, tb, fb, o, x_lengths=lens, f0_lengths=fl)
    ap = w.d4c(xb, FS, tb, fb, fft, x_lengths=lens, f0_lengths=fl)
    w.synchronize()
    return to_np(sp), to_np(ap)


def _same(got, want, what):
    for name, a, b in zip(("CheapTrick", "D4C"), got, want):
        assert a.shape == b.shape and np.array_equal(a, b), f"{name}, {what}: differs from a fresh context's rows"


# A short batch draws at most (1024 + 513) * 300 numbers per utterance in CheapTrick, within the table a context starts
# with (2^20 draws), and (1201 + 4089) * 300 in D4C, past it; the long batch's CheapTrick draws up to
# (2048 + 1025) * 1500, past the table the short batch left (2^21 draws).
SHORT = (601, 3, 300, 1024)
LONG = (611, 2, 1500, 2048)


def check_growth(world, ref):
    short, long_ = _batch(*SHORT), _batch(*LONG)
    fresh = []
    for b in (short, long_):
        f = _fresh(world)
        try:
            fresh.append(_spectral(f, b))
        finally:
            f.close()
    want_s, want_l = fresh
    w = _fresh(world)
    try:
        _same(_spectral(w, short), want_s, "short batch first")
        _same(_spectral(w, long_), want_l, "long batch after the short one (the table grows)")
        _same(_spectral(w, short), want_s, "short batch after the long one")
        w.trim()                                                             # (b)
        _same(_spectral(w, short), want_s, "short batch after trim()")
        _same(_spectral(w, long_), want_l, "long batch after trim() and the short batch")
    finally:
        w.close()
    for b, (sp, ap) in ((short, want_s), (long_, want_l)):
        x, t, f, lens, fl, fft = b
        u = len(fl) - 1
        xu, tu, fu = x[u, :lens[u]], t[u, :fl[u]], f[u, :fl[u]]
        o = ref.cheaptrick_option(FS)
        o.fft_size = fft
        assert_close(sp[u, :fl[u]], ref.cheaptrick(xu, FS, tu, fu, o), f"CheapTrick fft {fft}")
        assert_close(ap[u, :fl[u]], ref.d4c(xu, FS, tu, fu, fft), f"D4C fft {fft}")


def check_lanes(world):
    """analyze_batch cut into four slices (two lanes: sibling contexts on their own streams, each with its own table)
    against one slice on the context itself"""
    from synth import synth_batch
    from world_b200 import api
    x = make(world, synth_batch(range(621, 627), FS, 4800).numpy())
    lens = [4800 - 331 * u for u in range(6)]
    opt = world.analysis_option(FS, api.F0_DIO_STONEMASK)
    outs = []
    for slices in (1, 4, 1):
        w = _fresh(world)
        try:
            with lane_slices(slices):
                outs.append([to_np(a) for a in w.analyze_batch(x, FS, opt, x_lengths=lens)[:4]])
            w.synchronize()
        finally:
            w.close()
    for k, name in enumerate(("time axis", "f0", "spectrogram", "aperiodicity")):
        assert np.array_equal(outs[1][k], outs[0][k]), f"analyze_batch {name}: two lanes differ from one"
        assert np.array_equal(outs[2][k], outs[0][k]), f"analyze_batch {name}: one lane differs between runs"


def _grown(world):
    """A fresh context whose table the long batch has grown"""
    w = _fresh(world)
    _spectral(w, _batch(*LONG))
    return w


def check_options_and_packed(world):
    """(d) on a context with a grown table and again after trim()"""
    w = _grown(world)
    try:
        for _ in range(2):
            so.check_groups(w, FS, 3200, 6)
            pk.check_equal(w, FS, 3200, 4, method="dio")
            w.trim()
    finally:
        w.close()


def check_synthesis_packed(world):
    """(e) on a context with a grown table and again after trim()"""
    w = _grown(world)
    try:
        for _ in range(2):
            ps.check_full(w, FS)
            tp.check_equal(w, FS, 3200, 4, method="dio")
            w.trim()
    finally:
        w.close()


# ---------------------------------------------------------------- emulation (CPU suite)
def test_emu_randn_table_growth(emu, ref):
    check_growth(emu, ref)


def test_emu_randn_table_lanes(emu):
    check_lanes(emu)


def test_emu_randn_table_options_and_packed(emu):
    check_options_and_packed(emu)


def test_emu_randn_table_synthesis_packed(emu):
    check_synthesis_packed(emu)


# ---------------------------------------------------------------- CUDA library
@pytest.mark.gpu
def test_gpu_randn_table_growth(gpu_world, ref):
    check_growth(gpu_world, ref)


@pytest.mark.gpu
def test_gpu_randn_table_lanes(gpu_world):
    check_lanes(gpu_world)


@pytest.mark.gpu
def test_gpu_randn_table_options_and_packed(gpu_world):
    check_options_and_packed(gpu_world)


@pytest.mark.gpu
def test_gpu_randn_table_synthesis_packed(gpu_world):
    check_synthesis_packed(gpu_world)
