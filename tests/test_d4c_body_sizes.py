"""D4C's fast body kernel at the transform sizes it is compiled for, on the host emulation (CPU suite) and on the CUDA
library (-m gpu): rows against the reference's D4C on the reference's own f0; an f0 ramp that crosses the fast / slow
split; a ragged batch with unvoiced frames, cut into chunks at a small scratch budget, equal bit for bit
to the one-pass rows; the coded rows."""
import numpy as np
import pytest

from test_parity_common import assert_close, assert_close_signed, make, to_np
from test_stage_paths import SMALL_BUDGET, _contours, _same, _with_budget, f0_ramp

# rate -> d_fft of D4C (d4c.cpp:350-352): 2^(1 + int(log2(4 fs / 47 + 1))).  d_fft 512 (fs below ~6 kHz) is not
# checked: there the reference's band count (fs / 2 - 3000) / 3000 is negative and its D4C corrupts its own heap.
RATES = {8000: 1024, 11025: 1024, 16000: 2048, 24000: 2048, 32000: 4096, 48000: 4096}


def d4c_fft_size(fs):
    return int(2.0 ** (1 + int(np.log(4.0 * fs / 47.0 + 1) / np.log(2.0))))


def d4c_scratch_per_utt(fs, frames):
    """bytes of d4c_run's scratch per utterance (draws of pass A and B + per-frame slots)"""
    max_a = 2 * int(3.0 * fs / 40.0 / 2.0 + 0.5) + 1
    max_b = 3 * (2 * int(4.0 * fs / 47.0 / 2.0 + 0.5) + 1)
    return (max_a + max_b) * 4 * frames + 28 * frames + 64


def check_body_size(world, ref, fs):
    from synth import synth_batch
    assert d4c_fft_size(fs) == RATES[fs]
    fft = world.cheaptrick_option(fs).fft_size
    n_ap = ref.number_of_aperiodicities(fs)
    # Below 12 kHz D4C has no 3 kHz band, and there the library's rows do not follow the reference's (already so
    # before the body kernel was specialised by size); those rates check the chunked rows only.
    vs_ref = n_ap > 0

    # 1. rows against the reference on the reference's f0
    if vs_ref:
        x1 = synth_batch([701], fs, int(0.6 * fs)).numpy()
        tr, fr = ref.harvest(x1[0], fs)
        assert (fr > 0).sum() > 20
        ap = world.d4c(make(world, x1), fs, make(world, tr[None]), make(world, fr[None]), fft)
        world.synchronize()
        assert_close(to_np(ap)[0], ref.d4c(x1[0], fs, tr, fr, fft), f"D4C fs {fs}, reference f0")

    # 2. an f0 ramp across the fast / slow split (the slow side begins between 54 Hz at 16 kHz and 75 Hz at 48 kHz),
    # and its coded rows (CodeAperiodicity: nothing below 12 kHz)
    ramp = f0_ramp(fs)[::4].copy()
    ramp[::23] = 0.0
    n2 = int((len(ramp) - 1) * fs / 1000.0) + fs // 50
    x2 = synth_batch([702], fs, n2).numpy()
    t2 = np.arange(len(ramp)) / 1000.0
    xb, tb, fb = make(world, x2), make(world, t2[None]), make(world, ramp[None])
    assert (n_ap == 0) == (fs < 12000)
    ap = world.d4c(xb, fs, tb, fb, fft)
    world.synchronize()
    if vs_ref:
        cap = world.d4c_coded(xb, fs, tb, fb, fft)
        world.synchronize()
        want2 = ref.d4c(x2[0], fs, t2, ramp, fft)
        assert_close(to_np(ap)[0], want2, f"D4C fs {fs}, f0 ramp")
        assert_close_signed(to_np(cap)[0], ref.code_aperiodicity(want2, fs, fft), f"coded D4C fs {fs}, f0 ramp")

    # 3. a ragged batch with unvoiced frames: one pass against chunks
    n3 = int(0.5 * fs)
    fit = SMALL_BUDGET // d4c_scratch_per_utt(fs, int(1000.0 * n3 / fs) + 1)
    n_utt = max(3, fit + 1)                       # at least two passes at the small budget
    lens = [n3 - (n3 // (2 * n_utt)) * u for u in range(n_utt)]
    frames = [int(1000.0 * l / fs) + 1 for l in lens]
    x3 = synth_batch(range(711, 711 + n_utt), fs, n3).numpy()
    t3, f3 = _contours(np.random.default_rng(fs + 7), frames, frames[0])
    xb, tb, fb = make(world, x3), make(world, t3), make(world, f3)
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs = []
        for w in (world, small):
            outs.append(w.d4c(xb, fs, tb, fb, fft, x_lengths=lens, f0_lengths=frames))
            w.synchronize()
    finally:
        small.close()
    _same(outs[1], outs[0], f"D4C fs {fs}")
    one = to_np(outs[0])
    default = 1.0 - 1e-12                         # the row of an unvoiced or rejected frame
    analysed = [(one[u, :frames[u]] != default).any(axis=1) for u in range(n_utt)]
    assert sum(a.sum() for a in analysed) > 0
    if vs_ref:
        u = n_utt - 1
        want3 = ref.d4c(x3[u, :lens[u]], fs, t3[u, :frames[u]], f3[u, :frames[u]], fft)
        assert_close(one[u, :frames[u]], want3, f"D4C fs {fs}, ragged batch, last utterance")


@pytest.mark.parametrize("fs", list(RATES))
def test_emu_d4c_body_size(emu, ref, fs):
    check_body_size(emu, ref, fs)


@pytest.mark.gpu
@pytest.mark.parametrize("fs", list(RATES))
def test_gpu_d4c_body_size(gpu_world, ref, fs):
    check_body_size(gpu_world, ref, fs)
