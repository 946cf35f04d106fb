"""Pitch and formant curves (world_b200_modify_curves*, world_b200_transform_*packed_curves) on the CUDA library: the
checks of the host emulation, with each frame's envelope held to the reference within 1e-12 relative (the device's log
/ exp against the host's libm)."""
import pytest

import modify_curves_common as mcc


@pytest.mark.gpu
def test_gpu_modify_curves_constant_equals_factors(gpu_world):
    mcc.check_constant_equals_factors(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_curves_frames_equal_lone_calls(gpu_world, golden):
    mcc.check_frames_equal_lone_calls(gpu_world, golden)


@pytest.mark.gpu
def test_gpu_modify_curves_vs_reference(gpu_world, ref, golden):
    print(f"worst {mcc.check_vs_reference(gpu_world, ref, golden, exact=False):.2e} relative")


@pytest.mark.gpu
def test_gpu_modify_curves_null_halves(gpu_world):
    mcc.check_null_halves(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_curves_invalid(gpu_world):
    mcc.check_invalid(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_curves_transform_equals_stepwise(gpu_world):
    mcc.check_transform_equals_stepwise(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_curves_transform_constant_equals_factors(gpu_world):
    mcc.check_transform_constant_equals_factors(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_curves_transform_invalid(gpu_world):
    mcc.check_transform_invalid(gpu_world)
