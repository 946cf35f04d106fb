"""The way back on packed rows on the single-thread host emulation of the kernel sources (CPU): bit for bit the padded
calls, the round trip from packed analysis, passes, a relaid pass, edges, the reference and the EINVAL rules."""
import pytest

import packed_synthesis_common as ps


def test_emu_packed_synthesis_full(emu):
    ps.check_full(emu, 16000)


@pytest.mark.parametrize("family", ["coded", "pcm16", "scaled", "modified"])
def test_emu_packed_synthesis_coded(emu, family):
    ps.check_coded(emu, 16000, families=(family,))


def test_emu_packed_synthesis_host(emu):
    ps.check_host(emu)


def test_emu_packed_modify(emu):
    ps.check_modify(emu)


def test_emu_packed_round_trip(emu):
    ps.check_round_trip(emu)


def test_emu_packed_synthesis_long_among_short(emu):
    """A 1 s utterance among thirty of 0.05 s at the smallest budget."""
    ps.check_long_among_short(emu, 16000, 1.0, 0.05, 30, ps.SMALL_BUDGET)


def test_emu_packed_synthesis_relaid(emu):
    ps.check_relaid(emu)


def test_emu_packed_synthesis_edges(emu):
    ps.check_edges(emu)


def test_emu_packed_synthesis_vs_reference(emu, ref):
    ps.check_vs_ref(emu, ref)


def test_emu_packed_synthesis_invalid(emu):
    ps.check_invalid(emu)
