"""Synthesis from coded rows to 16-bit PCM (world_b200_synthesis_coded_batch_pcm16) and the pipelined host call
(world_b200_synthesis_coded_host) on the CUDA library: the checks of the host emulation over every rate / frame period /
dimension combination, pinned and pageable host buffers, and torch streams."""
import numpy as np
import pytest

import coded_synthesis_common as cs
import synthesis_host_common as sh
import test_parity_common as pc


@pytest.mark.gpu
@pytest.mark.parametrize("dims", [40, 60])
@pytest.mark.parametrize("fp", [2.5, 5.0])
@pytest.mark.parametrize("fs", [16000, 22050, 48000])
def test_gpu_synthesis_pcm16_equals_quantised(gpu_world, fs, fp, dims, tmp_path):
    sh.check_pcm_equals_quantised(gpu_world, fs, fp, dims, tmp_path)


@pytest.mark.gpu
def test_gpu_synthesis_pcm16_clips(gpu_world):
    sh.check_pcm_clips(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_host_equals_device(gpu_world):
    sh.check_host_equals_device(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_host_pipeline_chunks(gpu_world, capfd, monkeypatch):
    sh.check_pipeline_chunks(gpu_world, capfd, monkeypatch)


@pytest.mark.gpu
def test_gpu_synthesis_host_high_f0(gpu_world):
    sh.check_host_high_f0(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_pcm16_vs_reference(gpu_world, ref, golden):
    print(f"worst {sh.check_vs_reference(gpu_world, ref, golden)} LSB")


@pytest.mark.gpu
def test_gpu_synthesis_host_no_bands(gpu_world):
    sh.check_no_bands(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_host_invalid(gpu_world):
    sh.check_invalid(gpu_world)


@pytest.mark.gpu
def test_gpu_synthesis_host_pinned_and_pageable(gpu_world):
    """Pinned inputs and outputs (copies under the kernels) and pageable ones give identical results, in several
    chunks so that the copies of one chunk meet the kernels of another."""
    import torch
    from test_stage_paths import SMALL_BUDGET, _with_budget
    w, fs, fp, dims = gpu_world, 16000, 5.0, 60
    f0, csp, cap, fl, lens = cs.analysed_rows(w, fs, fp, dims, seeds=(381, 382, 383))
    yl = cs.ragged_y(fs, lens)
    Y, fft = max(yl), w.cheaptrick_option(fs).fft_size
    pinned = [torch.from_numpy(a).pin_memory() for a in (f0, csp, cap)]
    small = _with_budget(w, SMALL_BUDGET)
    try:
        for world in (w, small):
            for nbit, dt in ((16, torch.int16), (0, torch.float64)):
                want = world.synthesis_coded_host(f0, csp, cap, fft, fp, fs, Y, nbit=nbit, f0_lengths=fl, y_lengths=yl)
                out = torch.full((3, Y), 5, dtype=dt).pin_memory()
                got = world.synthesis_coded_host(*pinned, fft, fp, fs, Y, nbit=nbit, f0_lengths=fl, y_lengths=yl,
                                                 out=out)
                assert np.array_equal(got, want) and np.array_equal(out.numpy(), want)
                assert np.abs(want[0, :yl[0]]).max() > 0
    finally:
        small.close()


@pytest.mark.gpu
def test_gpu_synthesis_pcm16_on_a_side_stream(gpu_world):
    """The int16 device call with work enqueued on a non-default torch stream: the output lives on the input's device
    and equals the default stream's call."""
    import torch
    w, fs, fp, dims = gpu_world, 16000, 5.0, 40
    f0, csp, cap, fl, lens = cs.analysed_rows(w, fs, fp, dims, seeds=(391, 392, 393))
    fft = w.cheaptrick_option(fs).fft_size
    yl = cs.ragged_y(fs, lens)
    F, S, A = pc.make(w, f0), pc.make(w, csp), pc.make(w, cap)
    want = w.synthesis_coded(F, S, A, fft, fp, fs, max(yl), f0_lengths=fl, y_lengths=yl, dtype=torch.int16)
    w.synchronize()
    side = torch.cuda.Stream(device=0)
    side.wait_stream(torch.cuda.current_stream(0))
    with torch.cuda.stream(side):
        got = w.synthesis_coded(F, S, A, fft, fp, fs, max(yl), f0_lengths=fl, y_lengths=yl, dtype=torch.int16)
        done = got.to(torch.int64).sum()   # consumed on the same stream
    side.synchronize()
    torch.cuda.current_stream(0).wait_stream(side)
    assert got.device == F.device and got.dtype == torch.int16
    assert torch.equal(want, got) and int(done) == int(want.to(torch.int64).sum())
    assert int(got.abs().max()) > 30
    w._use_current_stream()   # back to the default stream for the tests that follow
