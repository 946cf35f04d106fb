"""CheapTrick and D4C with one option per utterance on the CUDA library: mixed FFT sizes at 16 / 22.05 / 48 kHz
against the reference, equal options against the one-option calls, size groups cut into scratch chunks."""
import pytest

import spectral_options_common as so

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000), (22050, 13230), (48000, 24000)]


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_spectral_options_vs_reference(gpu_world, ref, fs, n):
    so.check_vs_ref(gpu_world, ref, fs, n, n_utts=8, dims=60)


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_spectral_options_identity(gpu_world, fs, n):
    so.check_identity(gpu_world, fs, n)


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_spectral_options_groups(gpu_world, fs, n):
    so.check_groups(gpu_world, fs, n, 10)


def test_gpu_spectral_options_groups_in_chunks(gpu_world):
    """At 48 kHz a 2 s utterance at fft_size 4096 needs about 10 MB of CheapTrick draws, so the smallest budget runs
    each size group in chunks of a few utterances."""
    so.check_groups(gpu_world, 48000, 96000, 16, small_budget=True)


def test_gpu_spectral_options_layout(gpu_world):
    so.check_layout(gpu_world, 48000, 24000)


def test_gpu_spectral_options_invalid(gpu_world):
    so.check_invalid(gpu_world)


@pytest.mark.parametrize("fs,n", [(16000, 24000), (48000, 48000)])
def test_gpu_spectral_options_chain(gpu_world, fs, n):
    """Nine utterances in two lane slices."""
    so.check_chain(gpu_world, fs, n, 9, dims=60)
