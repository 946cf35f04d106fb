"""DIO at the rates, speeds and floors where its band sweep meets few events per tile, on voices that start or end
abruptly, on the single-thread host emulation of the kernel sources (CPU).  48 kHz is slow here: the grid is cut to
the cases that matter most; tests/test_gpu_dio_rate_edges.py runs all of it."""
import pytest

import dio_rate_edges_common as de

# (fs, speed, f0_ceil): undecimated 48 and 44.1 kHz at both ceilings, decimated 48 kHz, and the low rates as controls
CASES = [(48000, 1, 800.0), (48000, 1, 1100.0), (44100, 1, 800.0), (48000, 2, 800.0), (48000, 4, 1100.0),
         (32000, 1, 800.0), (16000, 1, 1100.0), (22050, 2, 800.0)]


@pytest.mark.parametrize("fs,speed,ceil", CASES)
def test_emu_dio_rate_edges_vs_reference(emu, ref, fs, speed, ceil):
    de.check_vs_ref(emu, ref, fs, speed, ceil)


@pytest.mark.parametrize("fs,speed", [(48000, 1), (44100, 1)])
def test_emu_dio_rate_edges_lone_call(emu, fs, speed):
    de.check_lone(emu, fs, speed)


def test_emu_dio_rate_edges_poisoned_scratch(emu):
    de.check_poison(emu)
