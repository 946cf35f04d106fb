"""Pitch and formant curves (world_b200_modify_curves*, world_b200_transform_*packed_curves) on the single-thread host
emulation of the kernel sources (CPU).  The emulation evaluates log / exp with the host's libm, as the restatement
does, so each frame's envelope is held to the reference bit for bit."""
import modify_curves_common as mcc


def test_emu_modify_curves_constant_equals_factors(emu):
    mcc.check_constant_equals_factors(emu)


def test_emu_modify_curves_frames_equal_lone_calls(emu, golden):
    mcc.check_frames_equal_lone_calls(emu, golden)


def test_emu_modify_curves_vs_reference(emu, ref, golden):
    mcc.check_vs_reference(emu, ref, golden, exact=True)


def test_emu_modify_curves_null_halves(emu):
    mcc.check_null_halves(emu)


def test_emu_modify_curves_invalid(emu):
    mcc.check_invalid(emu)


def test_emu_modify_curves_transform_equals_stepwise(emu):
    mcc.check_transform_equals_stepwise(emu)


def test_emu_modify_curves_transform_constant_equals_factors(emu):
    mcc.check_transform_constant_equals_factors(emu)


def test_emu_modify_curves_transform_invalid(emu):
    mcc.check_transform_invalid(emu)
