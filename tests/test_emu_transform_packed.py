"""The packed voice transformation on the single-thread host emulation of the kernel sources (CPU): every utterance's
samples equal the padded transform's bit for bit, across input and output widths, factors, F0 methods and options,
slices, host chunks, edges and the EINVAL rules."""
import pytest

import transform_packed_common as tp


@pytest.mark.parametrize("method", ["harvest", "dio"])
@pytest.mark.parametrize("f0_options", [True, False])
def test_emu_transform_packed_equals_padded(emu, method, f0_options):
    tp.check_equal(emu, 16000, 3200, 5, method=method, f0_options=f0_options)


def test_emu_transform_packed_one_spectral_option(emu):
    tp.check_equal(emu, 16000, 3200, 4, spectral_options=False, combos=[(16, 16, "both"), (0, 0, "none")])


def test_emu_transform_packed_host(emu):
    tp.check_host(emu)


def test_emu_transform_packed_slices(emu):
    """Four 1.5 s utterances at fft_size 4096: two fit a slice at the smallest budget, four do not."""
    tp.check_slices(emu, 16000, 1.5, 4, 4096, one_per_slice=False)


def test_emu_transform_packed_one_per_slice(emu):
    """Three 2.6 s utterances at fft_size 4096: no two fit a slice at the smallest budget."""
    tp.check_slices(emu, 16000, 2.6, 3, 4096, one_per_slice=True)


def test_emu_transform_packed_long_among_short(emu):
    """A 6 s utterance among thirty of 0.05 s at fft_size 4096 and the smallest budget."""
    tp.check_long_among_short(emu, 16000, 96000, 800, 30, fft=4096)


def test_emu_transform_packed_relaid(emu):
    tp.check_relaid(emu)


def test_emu_transform_packed_edges(emu):
    tp.check_edges(emu)


def test_emu_transform_packed_samples(emu):
    tp.check_samples(emu)


def test_emu_transform_packed_invalid(emu):
    tp.check_invalid(emu)
