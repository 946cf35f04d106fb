"""F0 scaling and formant shift (world_b200_modify_batch, world_b200_synthesis_coded_*_modified) on the CUDA library:
the checks of the host emulation, with the envelope held to the reference within 1e-12 relative (the device's log /
exp against the host's libm), and the reference's own demo program against the library's chain."""
import os

import pytest

import modify_common as mc


@pytest.mark.gpu
def test_gpu_modify_golden_vs_reference(gpu_world, ref, golden):
    print(f"worst {mc.check_golden(gpu_world, ref, golden, exact=False):.2e} relative")


@pytest.mark.gpu
@pytest.mark.parametrize("fs,fft", [(16000, 512), (16000, 1024), (22050, 1024), (48000, 2048)])
def test_gpu_modify_analysed_vs_reference(gpu_world, ref, fs, fft):
    print(f"worst {mc.check_analysed(gpu_world, ref, fs, fft, exact=False):.2e} relative")


@pytest.mark.gpu
def test_gpu_modify_identity_and_bounds(gpu_world):
    mc.check_identity_and_bounds(gpu_world)


@pytest.mark.gpu
@pytest.mark.parametrize("fs,fp,dims", [(16000, 5.0, 60), (22050, 2.5, 40), (48000, 5.0, 60)])
def test_gpu_modify_fused_equals_stepwise(gpu_world, fs, fp, dims):
    mc.check_fused_equals_stepwise(gpu_world, fs, fp, dims)


@pytest.mark.gpu
def test_gpu_modify_small_budget(gpu_world):
    mc.check_small_budget(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_scaled_high_f0(gpu_world):
    mc.check_scaled_high_f0(gpu_world)


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [False, True])
def test_gpu_modify_host_equals_device(gpu_world, pinned):
    mc.check_host_equals_device(gpu_world, pinned=pinned)


@pytest.mark.gpu
def test_gpu_modify_invalid(gpu_world):
    mc.check_invalid(gpu_world)


@pytest.mark.gpu
def test_gpu_modify_matches_the_reference_demo(gpu_world, golden, tmp_path):
    if not os.path.exists(mc.REF_DEMO):
        pytest.skip("oracle/_ref/ref_demo missing: build() found no reference sources")
    mc.check_ref_demo(gpu_world, golden, str(tmp_path))
