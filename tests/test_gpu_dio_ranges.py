"""DIO with one option per utterance on the CUDA library: the stage call at 16 (speed 1, 3, 12) / 22.05 / 48 kHz, the
device chain (both lanes), the host pipeline, the coded host chain with either F0 method and the multi-GPU chain at one
rank."""
import numpy as np
import pytest

import dio_ranges_common as dr
import test_parity_common as pc
from refworld import rel_err
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST, WorldError

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000, 1, [201, 202, 203, 204, 205]), (16000, 12000, 3, [206, 207, 208, 209, 210]),
         (22050, 13230, 1, [211, 212, 213, 214, 215]), (16000, 12000, 12, [216, 217, 218, 219, 220]),
         (48000, 24000, 1, [221, 222, 223, 224, 225])]


@pytest.mark.parametrize("fs,n,speed,seeds", CASES)
def test_gpu_dio_ranges_vs_reference(gpu_world, ref, fs, n, speed, seeds):
    dr.check_mixed_vs_ref(gpu_world, ref, fs, n, seeds, speed)


@pytest.mark.parametrize("fs,n,speed,seeds", CASES)
def test_gpu_dio_ranges_composition(gpu_world, fs, n, speed, seeds):
    dr.check_composition(gpu_world, fs, n, seeds + [s + 50 for s in seeds], speed)


def test_gpu_dio_ranges_scratch_chunks(gpu_world):
    dr.check_scratch_chunks(gpu_world)


def test_gpu_dio_ranges_invalid_utterance(gpu_world):
    dr.check_invalid(gpu_world)


@pytest.mark.parametrize("f0_method", [F0_HARVEST, F0_DIO_STONEMASK])
def test_gpu_coded_host_per_utterance_options(gpu_world, f0_method):
    dr.check_coded_host(gpu_world, f0_method)


def _mixed_chain_batch(w, fs=16000, n_samples=16000, n=12):
    x, lens = dr.batch(fs, n_samples, range(231, 231 + n))
    rng = [dr.RANGES[u % len(dr.RANGES)] for u in range(n)]
    return x, lens, rng, dr.options(rng), w.analysis_option(fs, F0_DIO_STONEMASK)


def test_gpu_analyze_batch_dio_options_vs_reference_chain(gpu_world, ref):
    """Twelve utterances, five options, two lanes: each row against the reference's own chain (its Dio at the
    utterance's option feeding its StoneMask, CheapTrick and D4C); the host pipeline gives the same f0 and time rows."""
    w, fs = gpu_world, 16000
    x, lens, rng, opts, ao = _mixed_chain_batch(w, fs)
    t, f0, sp, ap, fl = w.analyze_batch(pc.make(w, x), fs, ao, x_lengths=lens, dio_options=opts)
    w.synchronize()
    t, f0, sp, ap = (pc.to_np(a) for a in (t, f0, sp, ap))
    for u in range(len(x)):
        xu = np.ascontiguousarray(x[u, :lens[u]])
        tr, frd = ref.dio(xu, fs, dr.ref_option(ref, rng[u]))
        frf = ref.stonemask(xu, fs, tr, frd)
        co = ref.cheaptrick_option(fs)
        spr = ref.cheaptrick(xu, fs, tr, frf, co)
        apr = ref.d4c(xu, fs, tr, frf, co.fft_size)
        L = fl[u]
        assert np.array_equal(t[u, :L], tr)
        assert not ((f0[u, :L] > 0) != (frf > 0)).any(), f"V/UV flip, utterance {u}"
        assert rel_err(f0[u, :L], frf).max() <= pc.TOL
        assert rel_err(sp[u, :L], spr).max() <= pc.TOL, f"spectrogram, utterance {u}"
        assert rel_err(ap[u, :L], apr).max() <= pc.TOL, f"aperiodicity, utterance {u}"
    th, fh, sph, aph, flh = w.analyze_host(np.ascontiguousarray(x), fs, ao, x_lengths=lens, dio_options=opts)
    assert flh == fl
    assert np.array_equal(fh, f0) and np.array_equal(th, t)
    assert rel_err(sph, sp).max() <= 1e-12 and rel_err(aph, ap).max() <= 1e-12
    with pytest.raises(WorldError, match="error 3"):   # a bad band list half way through the batch names its utterance
        bad = dr.options(rng)
        bad[7].f0_ceil = 10.0
        w.analyze_batch(pc.make(w, x), fs, ao, x_lengths=lens, dio_options=bad)
    assert "utterance 7)" in w.lib.world_b200_last_error(w._h).decode()


def test_gpu_analyze_batch_allgather_dio_options_one_rank(gpu_world):
    """The multi-GPU chain at one rank (the communicator of a single process) gives the device chain's arrays."""
    import torch
    w, fs = gpu_world, 16000
    try:
        uid = w.comm_unique_id()
    except WorldError:
        pytest.skip("NCCL is not available")
    x, lens, rng, opts, ao = _mixed_chain_batch(w, fs, n=6)
    xb = pc.make(w, x)
    t, f0, sp, ap, fl = w.analyze_batch(xb, fs, ao, x_lengths=lens, dio_options=opts)
    tg, f0g = torch.zeros_like(t), torch.zeros_like(f0)
    spg, apg = torch.zeros_like(sp), torch.zeros_like(ap)
    w.comm_init(1, 0, uid)
    try:
        w.analyze_batch_allgather(xb, fs, ao, tg, f0g, spg, apg, x_lengths=lens, dio_options=opts)
        w.synchronize()
    finally:
        w.comm_destroy()
    for a, b in ((t, tg), (f0, f0g), (sp, spg), (ap, apg)):
        assert torch.equal(a, b)
