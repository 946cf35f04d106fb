"""The packed stage calls on the single-thread host emulation of the kernel sources (CPU): bit for bit the padded
_options calls and the packed chains, the packed codec, ragged edge cases, bounds, the reference and the EINVAL rules."""
import pytest

import packed_common as pk
import packed_stages_common as ps


@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_emu_packed_stages_equal_padded(emu, method):
    ps.check_equal(emu, 16000, 3200, 4, method=method)


def test_emu_packed_stages_external_f0(emu):
    """An F0 at a 10 ms hop against the chain's 5 ms, with unvoiced frames and frames below CheapTrick's floor."""
    ps.check_equal(emu, 16000, 3200, 4, ext_hop=10.0)


@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_emu_packed_stages_composition(emu, method):
    ps.check_composition(emu, 16000, 3200, 4, method=method)


def test_emu_packed_codec(emu):
    ps.check_codec(emu, 16000, 3200, 4)


def test_emu_packed_stages_edges(emu):
    ps.check_edges(emu, 16000, 2400)


def test_emu_packed_stages_long_among_short(emu):
    """A 1 s utterance among 30 of 0.03 s at the smallest scratch budget."""
    ps.check_long_among_short(emu, 16000, 16000, 480, 30, pk.SMALL_BUDGET)


def test_emu_packed_stages_bounds(emu):
    ps.check_bounds(emu, 16000, 3200)


def test_emu_packed_stages_vs_reference(emu, ref):
    ps.check_vs_ref(emu, ref, 16000, 4000)


def test_emu_packed_stages_invalid(emu):
    ps.check_invalid(emu)
