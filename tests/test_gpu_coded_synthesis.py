"""Synthesis from coded rows (world_b200_synthesis_coded_batch) on the CUDA library: the checks of the host emulation
over every rate / frame period / dimension combination, and torch streams."""
import numpy as np
import pytest

import coded_synthesis_common as cs
import test_parity_common as pc


@pytest.mark.gpu
@pytest.mark.parametrize("dims", [40, 60])
@pytest.mark.parametrize("fp", [2.5, 5.0])
@pytest.mark.parametrize("fs", [16000, 22050, 48000])
def test_gpu_synthesis_coded_equals_two_step(gpu_world, fs, fp, dims):
    cs.check_equals_two_step(gpu_world, fs, fp, dims)


@pytest.mark.gpu
def test_gpu_synthesis_coded_vs_reference(gpu_world, ref, golden):
    print(f"worst {cs.check_vs_reference(gpu_world, ref, golden):.2e} of the peak")


@pytest.mark.gpu
def test_gpu_synthesis_coded_no_bands(gpu_world, ref):
    print(f"worst {cs.check_no_bands(gpu_world, ref):.2e} of the peak")


@pytest.mark.gpu
def test_gpu_synthesis_coded_small_budget(gpu_world):
    cs.check_small_budget(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_coded_high_f0(gpu_world):
    cs.check_high_f0(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_coded_invalid(gpu_world):
    cs.check_invalid(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_coded_on_a_side_stream(gpu_world):
    """Work enqueued on a non-default torch stream: the output lives on the input's device and equals the default
    stream's call."""
    import torch
    w, fs, fp, dims = gpu_world, 16000, 5.0, 40
    f0, csp, cap, fl, lens = cs.analysed_rows(w, fs, fp, dims, seeds=(341, 342, 343))
    fft = w.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    F, S, A = pc.make(w, f0), pc.make(w, csp), pc.make(w, cap)
    want = w.synthesis_coded(F, S, A, fft, fp, fs, max(yl), f0_lengths=fl, y_lengths=yl)
    w.synchronize()
    side = torch.cuda.Stream(device=0)
    side.wait_stream(torch.cuda.current_stream(0))
    with torch.cuda.stream(side):
        got = w.synthesis_coded(F, S, A, fft, fp, fs, max(yl), f0_lengths=fl, y_lengths=yl)
        done = got.sum()   # consumed on the same stream
    side.synchronize()
    torch.cuda.current_stream(0).wait_stream(side)
    assert got.device == F.device and got.dtype == torch.float64
    assert torch.equal(want, got) and float(done) == float(want.sum())
    assert np.abs(pc.to_np(got)).max() > 1e-4
    w._use_current_stream()   # back to the default stream for the tests that follow
