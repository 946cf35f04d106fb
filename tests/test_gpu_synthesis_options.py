"""Synthesis, modification and the voice transform with one fft_size per utterance on the H100: every row equals the
one-size call on that utterance alone, bit for bit, at 16 kHz (512 / 1024 / 2048) and 48 kHz (2048 / 4096); a few
utterances of each size against the reference's Synthesis at that size; the transform against the stepwise chain."""
import numpy as np
import pytest

import synthesis_options_common as so
import test_parity_common as pc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fs", [16000, 48000])
@pytest.mark.parametrize("family", so.FAMILIES)
def test_gpu_synthesis_options_rows(gpu_world, family, fs):
    so.check_family(gpu_world, fs, family, n=6, seconds=1.5)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_synthesis_options_relaid(gpu_world, fs):
    so.check_relaid(gpu_world, fs, seconds=1.0)


def test_gpu_synthesis_options_all_equal(gpu_world):
    so.check_all_equal(gpu_world, seconds=1.0)


def test_gpu_synthesis_options_small_budget(gpu_world):
    so.check_small_budget(gpu_world)


@pytest.mark.parametrize("host", [False, True])
def test_gpu_transform_spectral_options(gpu_world, host):
    so.check_transform(gpu_world, n=6, seconds=1.0, host=host)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_transform_spectral_options_stepwise(gpu_world, fs):
    so.check_transform_stepwise(gpu_world, fs=fs, n=6, seconds=1.0)


def test_gpu_synthesis_options_invalid(gpu_world):
    so.check_invalid(gpu_world)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_synthesis_options_vs_reference(gpu_world, ref, fs):
    """Two utterances of each size of a mixed full-row call against the reference's Synthesis at that size: within 1e-9
    of the waveform peak, the bound of every Synthesis test."""
    b = so.Batch(gpu_world, fs, so.sizes_of(gpu_world, fs, 6), 1.0, 24, seed=21)
    y = so.run_family(gpu_world, b, "full")
    checked = {}
    for u in range(b.n):
        if checked.get(b.sizes[u], 0) >= 2:
            continue
        f0, sp, ap, _, _ = b.one(u)
        yr = ref.synthesis(np.ascontiguousarray(f0[0]), np.ascontiguousarray(sp[0]), np.ascontiguousarray(ap[0]),
                           b.sizes[u], so.FP, fs, b.y_len[u])
        e = np.abs(y[u, :b.y_len[u]] - yr).max() / max(np.abs(yr).max(), 1e-300)
        assert e <= 1e-9, f"utterance {u} (fft_size {b.sizes[u]}): {e:.2e} of the peak"
        checked[b.sizes[u]] = checked.get(b.sizes[u], 0) + 1
    assert len(checked) == len(set(b.sizes))
