"""The packed analysis chains on the single-thread host emulation of the kernel sources (CPU): bit for bit the padded
chains, ragged edge cases, lane slices and host chunks, bounds, the reference and the EINVAL rules."""
import pytest

import packed_common as pk


@pytest.mark.parametrize("method", ["harvest", "dio"])
@pytest.mark.parametrize("f0_options", [True, False])
def test_emu_packed_equals_padded(emu, method, f0_options):
    pk.check_equal(emu, 16000, 3200, 5, method=method, f0_options=f0_options)


def test_emu_packed_one_spectral_option(emu):
    pk.check_equal(emu, 16000, 3200, 3, spectral_options=False)


def test_emu_packed_edges(emu):
    pk.check_edges(emu, 16000, 2400)


def test_emu_packed_long_among_short(emu):
    """A 2 s utterance among 140 of 0.03 s; the smallest budget keeps 16 MB for a slice's padded rows."""
    pk.check_long_among_short(emu, 16000, 32000, 480, 140, pk.SMALL_BUDGET)


def test_emu_packed_slices_and_chunks(emu):
    pk.check_slices_and_chunks(emu, 16000, 3200, 7)


def test_emu_packed_bounds(emu):
    pk.check_bounds(emu, 16000, 3200)


def test_emu_packed_vs_reference(emu, ref):
    pk.check_vs_ref(emu, ref, 16000, 4000)


def test_emu_packed_invalid(emu):
    pk.check_invalid(emu)
