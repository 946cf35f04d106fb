"""The packed voice transformation on the CUDA library: every utterance's samples equal the padded transform's bit for
bit at 16 / 22.05 / 48 kHz, one 30 s utterance among forty of 0.5 s, several slices and one utterance per slice, host
chunks from pinned and pageable memory, a relaid pass, edges and the EINVAL rules."""
import pytest

import transform_packed_common as tp

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000), (22050, 13230), (48000, 24000)]


@pytest.mark.parametrize("fs,n", CASES)
@pytest.mark.parametrize("method", ["harvest", "dio"])
@pytest.mark.parametrize("f0_options", [True, False])
def test_gpu_transform_packed_equals_padded(gpu_world, fs, n, method, f0_options):
    tp.check_equal(gpu_world, fs, n, 8, method=method, f0_options=f0_options)


def test_gpu_transform_packed_one_spectral_option(gpu_world):
    tp.check_equal(gpu_world, 48000, 24000, 6, spectral_options=False)


@pytest.mark.parametrize("pinned", [False, True])
def test_gpu_transform_packed_host(gpu_world, pinned):
    tp.check_host(gpu_world, 22050, 13230, 7, pinned=(pinned,))


def test_gpu_transform_packed_slices(gpu_world):
    """Six 1 s utterances at fft_size 4096: two fit a slice at the smallest budget, six do not."""
    tp.check_slices(gpu_world, 16000, 1.0, 6, 4096, one_per_slice=False)


def test_gpu_transform_packed_one_per_slice(gpu_world):
    """Five 2 s utterances at fft_size 4096: no two fit a slice at the smallest budget."""
    tp.check_slices(gpu_world, 16000, 2.0, 5, 4096, one_per_slice=True)


def test_gpu_transform_packed_long_among_short(gpu_world):
    """One 30 s utterance among forty of 0.5 s at 16 kHz and the smallest budget."""
    tp.check_long_among_short(gpu_world, 16000, 480000, 8000, 40)


def test_gpu_transform_packed_relaid(gpu_world):
    tp.check_relaid(gpu_world)


def test_gpu_transform_packed_edges(gpu_world):
    tp.check_edges(gpu_world)


def test_gpu_transform_packed_samples(gpu_world):
    tp.check_samples(gpu_world)


def test_gpu_transform_packed_invalid(gpu_world):
    tp.check_invalid(gpu_world)
