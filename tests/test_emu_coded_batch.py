"""The coded chain on device arrays (world_b200_analyze_coded_batch*), on the single-thread host emulation of the kernel
sources (CPU)."""
import pytest

import coded_batch_common as cb
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST


@pytest.mark.parametrize("nbit", [0, 16, 24])
@pytest.mark.parametrize("f0_method", [F0_DIO_STONEMASK, F0_HARVEST])
def test_emu_coded_batch_equals_coded_host(emu, f0_method, nbit):
    cb.check_equals_host(emu, f0_method, nbit)


@pytest.mark.parametrize("f0_method", [F0_DIO_STONEMASK, F0_HARVEST])
def test_emu_coded_batch_vs_two_step(emu, f0_method):
    cb.check_vs_two_step(emu, f0_method)


@pytest.mark.parametrize("f0_method", [F0_DIO_STONEMASK, F0_HARVEST])
def test_emu_coded_batch_per_utterance_options(emu, f0_method):
    cb.check_options(emu, f0_method)


def test_emu_coded_batch_null_outputs(emu):
    cb.check_null_outputs(emu)


def test_emu_coded_batch_invalid(emu):
    cb.check_invalid(emu)
