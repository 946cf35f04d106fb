"""Synthesis on constructed f0, envelope and aperiodicity rows and coded rows, on the CUDA library: three call forms bit
for bit, the reference sample by sample within 1e-9 of the local peak, NaN where the reference is NaN
(tests/synthesis_edges_common.py)."""
import pytest

import synthesis_edges_common as se

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    se.report()


@pytest.mark.parametrize("fs", se.RATES)
@pytest.mark.parametrize("family", list(se.FAMILIES))
def test_gpu_synthesis_edges(gpu_world, ref, family, fs):
    se.check_family(gpu_world, ref, family, fs)


@pytest.mark.parametrize("fs", [8000, 16000, 22050, 48000])
def test_gpu_synthesis_edges_coded(gpu_world, ref, fs):
    se.check_coded(gpu_world, ref, fs)
