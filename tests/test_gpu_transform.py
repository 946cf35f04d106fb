"""Voice transformation (world_b200_transform_batch / world_b200_transform_host) on the CUDA library: the checks of the
host emulation on larger batches, pinned and pageable host buffers, and the reference's own demo program."""
import os

import pytest

import modify_common as mc
import transform_common as tc


@pytest.mark.gpu
@pytest.mark.parametrize("fs,fft,method,nbit", [(16000, 1024, "harvest", 16), (16000, 1024, "dio", 0),
                                                (22050, 1024, "dio", 24), (22050, 1024, "harvest", 16),
                                                (48000, 2048, "harvest", 0), (48000, 2048, "dio", 16)])
def test_gpu_transform_equals_stepwise(gpu_world, fs, fft, method, nbit):
    tc.check_stepwise(gpu_world, fs, fft, method, nbit, seconds=1.2)


@pytest.mark.gpu
def test_gpu_transform_relaid_pass(gpu_world):
    tc.check_relaid_pass(gpu_world)


@pytest.mark.gpu
def test_gpu_transform_null_factors(gpu_world):
    tc.check_null_factors(gpu_world)


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_gpu_transform_per_utterance_options(gpu_world, method):
    tc.check_per_utterance_options(gpu_world, method)


@pytest.mark.gpu
def test_gpu_transform_small_budget(gpu_world):
    tc.check_small_budget(gpu_world, seconds=2.0, one_per_slice=True)


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [False, True])
def test_gpu_transform_host_equals_device(gpu_world, pinned):
    tc.check_host_equals_device(gpu_world, pinned=pinned)


@pytest.mark.gpu
def test_gpu_transform_invalid(gpu_world):
    tc.check_invalid(gpu_world)


@pytest.mark.gpu
def test_gpu_transform_time_scale_vs_reference(gpu_world, ref, golden):
    tc.check_time_scale_vs_reference(gpu_world, ref, golden)


@pytest.mark.gpu
def test_gpu_transform_matches_the_reference_demo(gpu_world, golden, tmp_path):
    if not os.path.exists(mc.REF_DEMO):
        pytest.skip("oracle/_ref/ref_demo missing: build() found no reference sources")
    tc.check_ref_demo(gpu_world, golden, str(tmp_path))
