"""The way back on packed rows on the CUDA library: bit for bit the padded calls at 16 / 22.05 / 48 kHz, the round trip
from packed analysis, one 30 s utterance among forty of 0.5 s, a relaid pass, edges, the reference and the EINVAL
rules."""
import pytest

import packed_synthesis_common as ps

pytestmark = pytest.mark.gpu

RATES = [16000, 22050, 48000]


@pytest.mark.parametrize("fs", RATES)
def test_gpu_packed_synthesis_full(gpu_world, fs):
    ps.check_full(gpu_world, fs)


@pytest.mark.parametrize("fs", RATES)
def test_gpu_packed_synthesis_coded(gpu_world, fs):
    ps.check_coded(gpu_world, fs)


def test_gpu_packed_synthesis_host(gpu_world):
    ps.check_host(gpu_world)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_packed_modify(gpu_world, fs):
    ps.check_modify(gpu_world, fs)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_packed_round_trip(gpu_world, fs):
    ps.check_round_trip(gpu_world, fs, n=6, n_samples=fs // 2)


def test_gpu_packed_synthesis_long_among_short(gpu_world):
    """One 30 s utterance among forty of 0.5 s at 16 kHz, at the smallest budget."""
    ps.check_long_among_short(gpu_world, 16000, 30.0, 0.5, 40, ps.SMALL_BUDGET)


def test_gpu_packed_synthesis_relaid(gpu_world):
    ps.check_relaid(gpu_world)


def test_gpu_packed_synthesis_edges(gpu_world):
    ps.check_edges(gpu_world)


@pytest.mark.parametrize("fs", [16000, 48000])
def test_gpu_packed_synthesis_vs_reference(gpu_world, ref, fs):
    ps.check_vs_ref(gpu_world, ref, fs)


def test_gpu_packed_synthesis_invalid(gpu_world):
    ps.check_invalid(gpu_world)
