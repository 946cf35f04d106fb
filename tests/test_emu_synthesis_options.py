"""Synthesis, modification and the voice transform with one fft_size per utterance, on the single-thread host
emulation of the kernel sources (CPU), at 16 kHz (sizes 512 / 1024 / 2048, interleaved)."""
import pytest

import synthesis_options_common as so


@pytest.mark.parametrize("family", so.FAMILIES)
def test_emu_synthesis_options_rows(emu, family):
    so.check_family(emu, 16000, family)


def test_emu_synthesis_options_relaid(emu):
    so.check_relaid(emu, 16000)


def test_emu_synthesis_options_all_equal(emu):
    so.check_all_equal(emu)


def test_emu_synthesis_options_small_budget(emu):
    so.check_small_budget(emu)


@pytest.mark.parametrize("host", [False, True])
def test_emu_transform_spectral_options(emu, host):
    so.check_transform(emu, host=host)


def test_emu_transform_spectral_options_stepwise(emu):
    so.check_transform_stepwise(emu)


def test_emu_synthesis_options_invalid(emu):
    so.check_invalid(emu)
