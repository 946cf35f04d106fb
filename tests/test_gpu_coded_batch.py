"""The coded chain on device arrays (world_b200_analyze_coded_batch*) on the CUDA library: the equality checks of the
host emulation, parity with the compiled reference, the one-rank gather and torch streams."""
import numpy as np
import pytest

import coded_batch_common as cb
import f0_ranges_common as hr
import test_parity_common as pc
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST, WorldError


@pytest.mark.gpu
@pytest.mark.parametrize("nbit", [0, 16, 24])
@pytest.mark.parametrize("f0_method", [F0_DIO_STONEMASK, F0_HARVEST])
def test_gpu_coded_batch_equals_coded_host(gpu_world, f0_method, nbit):
    cb.check_equals_host(gpu_world, f0_method, nbit)


@pytest.mark.gpu
@pytest.mark.parametrize("f0_method", [F0_DIO_STONEMASK, F0_HARVEST])
def test_gpu_coded_batch_vs_two_step(gpu_world, f0_method):
    cb.check_vs_two_step(gpu_world, f0_method)


@pytest.mark.gpu
@pytest.mark.parametrize("f0_method", [F0_DIO_STONEMASK, F0_HARVEST])
def test_gpu_coded_batch_per_utterance_options(gpu_world, f0_method):
    cb.check_options(gpu_world, f0_method)


@pytest.mark.gpu
def test_gpu_coded_batch_null_outputs(gpu_world):
    cb.check_null_outputs(gpu_world)


@pytest.mark.gpu
def test_gpu_coded_batch_invalid(gpu_world):
    cb.check_invalid(gpu_world)


@pytest.mark.gpu
@pytest.mark.parametrize("fs", [16000, 44100])
def test_gpu_coded_batch_vs_reference(gpu_world, ref, fs):
    """Harvest f0 and time axis against the reference's Harvest, and the coded rows against the reference's
    CodeSpectralEnvelope(CheapTrick(...)) / CodeAperiodicity(D4C(...)) on the f0 the chain produced, within 1e-6."""
    w = gpu_world
    x, lens = hr.ragged_batch(fs, fs // 2, [181, 182, 183])
    ao = w.analysis_option(fs, F0_HARVEST)
    fft, dims = ao.cheaptrick.fft_size, 60
    t, f0, csp, cap, fl = cb.coded_batch(w, np.ascontiguousarray(x), 0, fs, ao, dims=dims, lens=lens)
    n_ap = ref.number_of_aperiodicities(fs)
    for u in range(len(lens)):
        xu, L = x[u, :lens[u]], fl[u]
        tr, fr = ref.harvest(xu, fs)
        assert np.array_equal(t[u, :L], tr)
        pc.assert_close(f0[u, :L], fr, f"f0 utterance {u}")
        fu = np.ascontiguousarray(f0[u, :L])
        want_sp = ref.code_spectral_envelope(ref.cheaptrick(xu, fs, tr, fu), fs, fft, dims)
        want_ap = ref.code_aperiodicity(ref.d4c(xu, fs, tr, fu, fft), fs, fft)
        pc.assert_close_signed(csp[u, :L], want_sp, f"coded sp fs={fs} utterance {u}")
        pc.assert_close_signed(cap[u, :L, :n_ap], want_ap[:, :n_ap], f"coded ap fs={fs} utterance {u}")
        assert (fr > 0).sum() > 10


@pytest.mark.gpu
def test_gpu_coded_batch_allgather_one_rank(gpu_world):
    """The coded multi-GPU chain at one rank (the communicator of a single process) gives analyze_coded_batch's arrays,
    with and without per-utterance options."""
    import torch
    w, fs = gpu_world, 16000
    try:
        uid = w.comm_unique_id()
    except WorldError:
        pytest.skip("NCCL is not available")
    x, lens = hr.ragged_batch(fs, 8000, [191, 192, 193, 194, 195, 196])
    pcm = pc.make(w, cb.pcm_rows(0.5 * x, 16)[0], dtype=np.int16)
    ao = w.analysis_option(fs, F0_HARVEST)
    w.comm_init(1, 0, uid)   # (an NCCL id makes one communicator)
    try:
        for kw in ({}, cb.per_utt_options(F0_HARVEST, len(lens))):
            want = w.analyze_coded_batch(pcm, 16, fs, ao, cb.DIMS, x_lengths=lens, **kw)
            got = [torch.zeros_like(a) for a in want[:4]]
            w.analyze_coded_batch_allgather(pcm, 16, fs, ao, cb.DIMS, *got, x_lengths=lens, **kw)
            w.synchronize()
            for a, b in zip(want[:4], got):
                assert torch.equal(a, b)
    finally:
        w.comm_destroy()


@pytest.mark.gpu
def test_gpu_coded_batch_int16_on_a_side_stream(gpu_world):
    """int16 torch tensors in, work enqueued on a non-default torch stream: the outputs live on the input's device and
    equal the default stream's call."""
    import torch
    w, fs = gpu_world, 16000
    x, lens = hr.ragged_batch(fs, 8000, [201, 202, 203, 204])
    pcm = torch.from_numpy(cb.pcm_rows(0.5 * x, 16)[0]).to("cuda:0")
    assert pcm.dtype == torch.int16
    ao = w.analysis_option(fs, F0_DIO_STONEMASK)
    want = w.analyze_coded_batch(pcm, 16, fs, ao, cb.DIMS, x_lengths=lens)
    w.synchronize()
    side = torch.cuda.Stream(device=0)
    side.wait_stream(torch.cuda.current_stream(0))
    with torch.cuda.stream(side):
        got = w.analyze_coded_batch(pcm, 16, fs, ao, cb.DIMS, x_lengths=lens)
        done = [a.sum() for a in got[:4]]   # consumed on the same stream
    side.synchronize()
    torch.cuda.current_stream(0).wait_stream(side)
    for a, b, s in zip(want[:4], got[:4], done):
        assert b.device == pcm.device and b.dtype == torch.float64
        assert torch.equal(a, b) and float(s) == float(a.sum())
    w._use_current_stream()   # back to the default stream for the tests that follow
