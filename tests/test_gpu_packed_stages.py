"""The packed stage calls on the CUDA library: bit for bit the padded _options calls at 16 / 22.05 / 48 kHz with two
CheapTrick sizes per batch, on DIO's, Harvest's and an external F0; the packed chains' rows by composition; the packed
codec; ragged edge cases, one 30 s utterance among forty of 0.5 s at the smallest budget, bounds, the reference and
the EINVAL rules."""
import pytest

import packed_common as pk
import packed_stages_common as ps

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000), (22050, 13230), (48000, 24000)]


@pytest.mark.parametrize("fs,n", CASES)
@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_gpu_packed_stages_equal_padded(gpu_world, fs, n, method):
    ps.check_equal(gpu_world, fs, n, 8, method=method)


def test_gpu_packed_stages_above_48k(gpu_world):
    """At 50 kHz D4C's transform is 8192 points: every selected frame goes through the frame list."""
    ps.check_equal(gpu_world, 50000, 25000, 4)


def test_gpu_packed_stages_many_utterances(gpu_world):
    """70,000 utterances: two chunks of at most 65,535."""
    ps.check_many_utterances(gpu_world)


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_packed_stages_external_f0(gpu_world, fs, n):
    """An F0 at a 10 ms hop against the chain's 5 ms, with unvoiced frames and frames below CheapTrick's floor."""
    ps.check_equal(gpu_world, fs, n, 8, ext_hop=10.0)


@pytest.mark.parametrize("fs,n", CASES)
@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_gpu_packed_stages_composition(gpu_world, fs, n, method):
    ps.check_composition(gpu_world, fs, n, 6, method=method)


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_packed_codec(gpu_world, fs, n):
    ps.check_codec(gpu_world, fs, n, 6)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_packed_stages_edges(gpu_world, fs):
    ps.check_edges(gpu_world, fs, fs // 2)


def test_gpu_packed_stages_long_among_short(gpu_world):
    """One 30 s utterance among forty of 0.5 s at 16 kHz, at the smallest scratch budget."""
    ps.check_long_among_short(gpu_world, 16000, 480000, 8000, 40, pk.SMALL_BUDGET)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_packed_stages_bounds(gpu_world, fs):
    ps.check_bounds(gpu_world, fs, fs // 2)


@pytest.mark.parametrize("fs,n", CASES)
def test_gpu_packed_stages_vs_reference(gpu_world, ref, fs, n):
    ps.check_vs_ref(gpu_world, ref, fs, n)


def test_gpu_packed_stages_invalid(gpu_world):
    ps.check_invalid(gpu_world)
