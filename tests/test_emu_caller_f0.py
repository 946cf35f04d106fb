"""StoneMask, CheapTrick and D4C on constructed caller F0 and time axes, on the single-thread host emulation of the
kernel sources (CPU): three call forms bit for bit, the reference frame by frame, StoneMask against its long-double
restatement, the refused frames and poisoned scratch (tests/caller_f0_common.py)."""
import pytest

import caller_f0_common as cf


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    cf.report()


@pytest.mark.parametrize("fs", cf.RATES)
def test_emu_caller_f0_stonemask(emu, ref, fs):
    cf.check_stonemask(emu, ref, fs)


@pytest.mark.parametrize("fs", cf.RATES)
def test_emu_caller_f0_cheaptrick(emu, ref, fs):
    cf.check_cheaptrick(emu, ref, fs)


@pytest.mark.parametrize("fs", cf.RATES)
def test_emu_caller_f0_d4c(emu, ref, fs):
    cf.check_d4c(emu, ref, fs)


@pytest.mark.parametrize("fs", [8000, 16000, 48000])
def test_emu_caller_f0_refused(emu, fs):
    cf.check_refused(emu, fs)


def test_emu_caller_f0_poison(emu):
    cf.check_poison(emu, 22050)
