"""Synthesis from coded rows (world_b200_synthesis_coded_batch) on the single-thread host emulation of the kernel
sources (CPU)."""
import pytest

import coded_synthesis_common as cs


@pytest.mark.parametrize("fs,fp,dims", [(16000, 5.0, 60), (16000, 2.5, 40), (22050, 2.5, 60), (48000, 5.0, 40)])
def test_emu_synthesis_coded_equals_two_step(emu, fs, fp, dims):
    cs.check_equals_two_step(emu, fs, fp, dims)


def test_emu_synthesis_coded_vs_reference(emu, ref, golden):
    print(f"worst {cs.check_vs_reference(emu, ref, golden):.2e} of the peak")


def test_emu_synthesis_coded_no_bands(emu, ref):
    print(f"worst {cs.check_no_bands(emu, ref):.2e} of the peak")


def test_emu_synthesis_coded_small_budget(emu):
    cs.check_small_budget(emu)


def test_emu_synthesis_coded_high_f0(emu):
    cs.check_high_f0(emu)


def test_emu_synthesis_coded_invalid(emu):
    cs.check_invalid(emu)
