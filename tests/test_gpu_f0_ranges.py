"""Harvest with one F0 range per utterance on the CUDA library: the stage call at 16 / 22.05 / 48 kHz, the device
chain (both lanes), the host pipeline and the multi-GPU chain at one rank."""
import numpy as np
import pytest

import f0_ranges_common as fr
import test_parity_common as pc
from refworld import rel_err
from world_b200.api import WorldError

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000, [101, 102, 103, 104, 105]), (22050, 13230, [106, 107, 108, 109, 110]),
         (48000, 24000, [111, 112, 113, 114, 115])]


@pytest.mark.parametrize("fs,n,seeds", CASES)
def test_gpu_f0_ranges_vs_reference(gpu_world, ref, fs, n, seeds):
    fr.check_mixed_vs_ref(gpu_world, ref, fs, n, seeds)


@pytest.mark.parametrize("fs,n,seeds", CASES)
def test_gpu_f0_ranges_composition(gpu_world, fs, n, seeds):
    fr.check_composition(gpu_world, fs, n, seeds + [s + 50 for s in seeds])


def test_gpu_f0_ranges_invalid_utterance(gpu_world):
    fr.check_invalid_range(gpu_world, 16000)


def _mixed_chain_batch(w, fs=16000, n_samples=16000, n=12):
    x, lens = fr.ragged_batch(fs, n_samples, range(121, 121 + n))
    rng = [fr.RANGES[u % len(fr.RANGES)] for u in range(n)]
    return x, lens, rng, fr.options(rng), w.analysis_option(fs, 1)


def test_gpu_analyze_batch_options_vs_reference_chain(gpu_world, ref):
    """Twelve utterances, five ranges, two lanes: each checked row against the reference's own chain (its Harvest at
    the utterance's option feeding its CheapTrick and D4C); the host pipeline gives the same f0 rows."""
    w, fs = gpu_world, 16000
    x, lens, rng, opts, ao = _mixed_chain_batch(w, fs)
    t, f0, sp, ap, fl = w.analyze_batch(pc.make(w, x), fs, ao, x_lengths=lens, harvest_options=opts)
    w.synchronize()
    t, f0, sp, ap = (pc.to_np(a) for a in (t, f0, sp, ap))
    for u in range(len(x)):
        xu = np.ascontiguousarray(x[u, :lens[u]])
        ro = ref.harvest_option()
        ro.f0_floor, ro.f0_ceil = rng[u]
        tr, frf = ref.harvest(xu, fs, ro)
        co = ref.cheaptrick_option(fs)
        spr = ref.cheaptrick(xu, fs, tr, frf, co)
        apr = ref.d4c(xu, fs, tr, frf, co.fft_size)
        L = fl[u]
        assert np.array_equal(t[u, :L], tr)
        assert not ((f0[u, :L] > 0) != (frf > 0)).any(), f"V/UV flip, utterance {u}"
        assert rel_err(f0[u, :L], frf).max() <= pc.TOL
        assert rel_err(sp[u, :L], spr).max() <= pc.TOL, f"spectrogram, utterance {u}"
        assert rel_err(ap[u, :L], apr).max() <= pc.TOL, f"aperiodicity, utterance {u}"
    th, fh, sph, aph, flh = w.analyze_host(np.ascontiguousarray(x), fs, ao, x_lengths=lens, harvest_options=opts)
    assert flh == fl
    assert np.array_equal(fh, f0) and np.array_equal(th, t)
    assert rel_err(sph, sp).max() <= 1e-12 and rel_err(aph, ap).max() <= 1e-12
    with pytest.raises(WorldError, match="error 3"):   # a bad range half way through the batch names its utterance
        bad = fr.options(rng)
        bad[7].f0_floor = 8.0
        w.analyze_batch(pc.make(w, x), fs, ao, x_lengths=lens, harvest_options=bad)
    assert "utterance 7)" in w.lib.world_b200_last_error(w._h).decode()


def test_gpu_analyze_batch_allgather_options_one_rank(gpu_world):
    """The multi-GPU chain at one rank (the communicator of a single process) gives the device chain's arrays."""
    import torch
    w, fs = gpu_world, 16000
    try:
        uid = w.comm_unique_id()
    except WorldError:
        pytest.skip("NCCL is not available")
    x, lens, rng, opts, ao = _mixed_chain_batch(w, fs, n=6)
    xb = pc.make(w, x)
    t, f0, sp, ap, fl = w.analyze_batch(xb, fs, ao, x_lengths=lens, harvest_options=opts)
    tg, f0g = torch.zeros_like(t), torch.zeros_like(f0)
    spg, apg = torch.zeros_like(sp), torch.zeros_like(ap)
    w.comm_init(1, 0, uid)
    try:
        w.analyze_batch_allgather(xb, fs, ao, tg, f0g, spg, apg, x_lengths=lens, harvest_options=opts)
        w.synchronize()
    finally:
        w.comm_destroy()
    for a, b in ((t, tg), (f0, f0g), (sp, spg), (ap, apg)):
        assert torch.equal(a, b)
