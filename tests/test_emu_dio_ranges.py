"""DIO with one option per utterance, and the coded host chain with per-utterance options of either F0 method, on the
single-thread host emulation of the kernel sources (CPU)."""
import pytest

import dio_ranges_common as dr
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST

# 16 kHz at speed 12 decimates to 1333 Hz: the 40-1100 Hz list has bands above afs / 2 (all-zero filters)
CASES = [(16000, 8000, 1, [81, 82, 83, 84, 85]), (16000, 8000, 3, [86, 87, 88, 89, 90]),
         (22050, 8820, 1, [91, 92, 93, 94, 95]), (16000, 8000, 12, [96, 97, 98, 99, 100])]


@pytest.mark.parametrize("fs,n,speed,seeds", CASES)
def test_emu_dio_ranges_vs_reference(emu, ref, fs, n, speed, seeds):
    dr.check_mixed_vs_ref(emu, ref, fs, n, seeds, speed)


@pytest.mark.parametrize("speed", [1, 12])
def test_emu_dio_ranges_composition(emu, speed):
    dr.check_composition(emu, 16000, 8000, [101, 102, 103, 104, 105, 106, 107], speed)


def test_emu_dio_ranges_scratch_chunks(emu):
    dr.check_scratch_chunks(emu)


def test_emu_dio_ranges_invalid_utterance(emu):
    dr.check_invalid(emu)


@pytest.mark.parametrize("f0_method", [F0_HARVEST, F0_DIO_STONEMASK])
def test_emu_coded_host_per_utterance_options(emu, f0_method):
    dr.check_coded_host(emu, f0_method)
