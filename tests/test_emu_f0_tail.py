"""The F0 decision stages (Harvest after candidate refinement, DIO's contour) on constructed candidate maps against
the reference's own functions, on the single-thread host emulation of the kernel sources (CPU)."""
import f0_tail_common as ft
from f0_tail_common import tail  # noqa: F401  (fixture)


def test_emu_f0_tail_wrapper_pin(emu, ref, tail, golden):
    ft.check_wrapper_pin(emu, ref, tail, golden)


def test_emu_f0_tail_merge(emu, tail):
    ft.check_merge(emu, tail)


def test_emu_f0_tail_extend(emu, tail):
    ft.check_extend(emu, tail)


def test_emu_f0_tail_ties_and_counts(emu, tail):
    ft.check_ties_and_counts(emu, tail)


def test_emu_f0_tail_frame_periods(emu, tail):
    ft.check_frame_periods(emu, tail)


def test_emu_f0_tail_ragged_batch(emu, tail):
    ft.check_ragged_batch(emu, tail)


def test_emu_f0_tail_dense_sections(emu, tail):
    ft.check_dense(emu, tail)


def test_emu_f0_tail_random(emu, tail):
    rep = ft.check_random(emu, tail, 300, seed=1)
    assert rep.maps == 300 and rep.sections > 3000 and rep.merged > 1500, rep


def test_emu_f0_tail_load_errors(emu, tail):
    ft.check_load_errors(emu, tail)


def test_emu_f0_tail_dio(emu, tail):
    ft.check_dio(emu, tail)
