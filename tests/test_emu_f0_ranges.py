"""Harvest with one F0 range per utterance, on the single-thread host emulation of the kernel sources (CPU)."""
import pytest

import f0_ranges_common as fr


@pytest.mark.parametrize("fs,n,seeds", [(16000, 8000, [81, 82, 83, 84]), (22050, 8820, [85, 86, 87, 88])])
def test_emu_f0_ranges_vs_reference(emu, ref, fs, n, seeds):
    fr.check_mixed_vs_ref(emu, ref, fs, n, seeds)


def test_emu_f0_ranges_composition(emu):
    fr.check_composition(emu, 16000, 8000, [91, 92, 93, 94, 95, 96])


def test_emu_f0_ranges_invalid_utterance(emu):
    fr.check_invalid_range(emu, 16000)
