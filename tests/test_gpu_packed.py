"""The packed analysis chains on the CUDA library: bit for bit the padded chains at 16 / 22.05 / 48 kHz, ragged edge
cases, one 30 s utterance among 0.5 s ones, lane slices and host chunks, bounds, the reference and the EINVAL rules."""
import pytest

import packed_common as pk

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000), (22050, 13230), (48000, 24000)]


@pytest.mark.parametrize("fs,n", CASES)
@pytest.mark.parametrize("method", ["harvest", "dio"])
@pytest.mark.parametrize("f0_options", [True, False])
def test_gpu_packed_equals_padded(gpu_world, fs, n, method, f0_options):
    pk.check_equal(gpu_world, fs, n, 10, method=method, f0_options=f0_options)


def test_gpu_packed_one_spectral_option(gpu_world):
    pk.check_equal(gpu_world, 48000, 24000, 6, spectral_options=False)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_packed_edges(gpu_world, fs):
    pk.check_edges(gpu_world, fs, fs // 2)


def test_gpu_packed_long_among_short(gpu_world):
    """One 30 s utterance among forty of 0.5 s at 16 kHz; the smallest budget keeps 16 MB for a slice's padded rows."""
    pk.check_long_among_short(gpu_world, 16000, 480000, 8000, 40, pk.SMALL_BUDGET)


def test_gpu_packed_slices_and_chunks(gpu_world):
    pk.check_slices_and_chunks(gpu_world, 48000, 96000, 11)


def test_gpu_packed_bounds(gpu_world):
    pk.check_bounds(gpu_world, 48000, 24000)


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_packed_vs_reference(gpu_world, ref, fs, n):
    pk.check_vs_ref(gpu_world, ref, fs, n)


def test_gpu_packed_invalid(gpu_world):
    pk.check_invalid(gpu_world)
