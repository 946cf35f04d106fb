"""StoneMask, CheapTrick and D4C on constructed caller F0 and time axes, on the CUDA library: three call forms bit for
bit, the reference frame by frame, StoneMask against its long-double restatement, the refused frames and poisoned scratch (tests/caller_f0_common.py)."""
import pytest

import caller_f0_common as cf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    cf.report()


@pytest.mark.parametrize("fs", cf.RATES)
def test_gpu_caller_f0_stonemask(gpu_world, ref, fs):
    cf.check_stonemask(gpu_world, ref, fs)


@pytest.mark.parametrize("fs", cf.RATES)
def test_gpu_caller_f0_cheaptrick(gpu_world, ref, fs):
    cf.check_cheaptrick(gpu_world, ref, fs)


@pytest.mark.parametrize("fs", cf.RATES)
def test_gpu_caller_f0_d4c(gpu_world, ref, fs):
    cf.check_d4c(gpu_world, ref, fs)


@pytest.mark.parametrize("fs", [8000, 16000, 48000])
def test_gpu_caller_f0_refused(gpu_world, fs):
    cf.check_refused(gpu_world, fs)


def test_gpu_caller_f0_poison(gpu_world):
    cf.check_poison(gpu_world, 22050)
