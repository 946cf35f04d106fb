"""CheapTrick and D4C with one option per utterance, on the single-thread host emulation of the kernel sources
(CPU)."""
import pytest

import spectral_options_common as so


@pytest.mark.parametrize("fs,n", [(16000, 4000), (22050, 4410)])
def test_emu_spectral_options_vs_reference(emu, ref, fs, n):
    so.check_vs_ref(emu, ref, fs, n)


def test_emu_spectral_options_identity(emu):
    so.check_identity(emu, 16000, 3200)


def test_emu_spectral_options_groups(emu):
    so.check_groups(emu, 16000, 3200, 6)


def test_emu_spectral_options_layout(emu):
    so.check_layout(emu, 16000, 3200)


def test_emu_spectral_options_invalid(emu):
    so.check_invalid(emu)


def test_emu_spectral_options_chain(emu):
    so.check_chain(emu, 16000, 4000, 4)
