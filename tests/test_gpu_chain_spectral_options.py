"""The full-row analysis chains with one CheapTrick / D4C option per utterance on the CUDA library: each speaker's
group at 16 / 22.05 / 48 kHz, the padded layout, equal options, the reference, lane slices and host chunks, the EINVAL
rules, and both new all-gather calls at one rank."""
import numpy as np
import pytest

import chain_spectral_options_common as cs
import test_parity_common as pc
from world_b200.api import WorldError

pytestmark = pytest.mark.gpu

CASES = [(16000, 12000), (22050, 13230), (48000, 24000)]


@pytest.mark.parametrize("fs,n", CASES)
@pytest.mark.parametrize("method", ["harvest", "dio"])
@pytest.mark.parametrize("f0_options", [True, False])
def test_gpu_chain_spectral_options_groups(gpu_world, fs, n, method, f0_options):
    """Ten utterances in two lane slices."""
    cs.check_groups(gpu_world, fs, n, 10, method=method, f0_options=f0_options)


def test_gpu_chain_spectral_options_layout(gpu_world):
    cs.check_layout(gpu_world, 48000, 24000)


@pytest.mark.parametrize("fs,n", [(16000, 12000), (48000, 24000)])
@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_gpu_chain_spectral_options_identity(gpu_world, fs, n, method):
    cs.check_identity(gpu_world, fs, n, method=method)


@pytest.mark.parametrize("fs,n", CASES)
@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_gpu_chain_spectral_options_vs_reference(gpu_world, ref, fs, n, method):
    cs.check_vs_ref(gpu_world, ref, fs, n, n_utts=8, method=method)


def test_gpu_chain_spectral_options_slices_and_chunks(gpu_world):
    """At 48 kHz a 2 s utterance at fft_size 4096 needs about 10 MB of CheapTrick draws, so the smallest budget runs
    each size group in chunks of a few utterances."""
    cs.check_slices_and_chunks(gpu_world, 48000, 96000, 11)


def test_gpu_chain_spectral_options_invalid(gpu_world):
    cs.check_invalid(gpu_world)


def test_gpu_chain_spectral_options_allgather_one_rank(gpu_world):
    """Both new all-gather calls under the communicator of a single process give the device chains' arrays."""
    import torch
    w, fs, dims = gpu_world, 48000, 60
    try:
        uid = w.comm_unique_id()
    except WorldError:
        pytest.skip("NCCL is not available")
    c = cs.Case(w, fs, 24000, 9)
    xb = pc.make(w, c.x)
    kw = dict(x_lengths=c.lens, **c.kw)
    t, f0, sp, ap, _ = w.analyze_batch(xb, fs, c.ao, **kw)
    ct, cf0, csp, cap, _ = w.analyze_coded_batch(xb, 0, fs, c.ao, dims, **kw)
    full = [torch.zeros_like(a) for a in (t, f0, sp, ap)]
    coded = [torch.zeros_like(a) for a in (ct, cf0, csp, cap)]
    w.comm_init(1, 0, uid)
    try:
        w.analyze_batch_allgather(xb, fs, c.ao, *full, **kw)
        w.analyze_coded_batch_allgather(xb, 0, fs, c.ao, dims, *coded, **kw)
        w.synchronize()
    finally:
        w.comm_destroy()
    assert sp.shape[-1] == c.width
    for name, a, b in zip(("t", "f0", "sp", "ap", "coded t", "coded f0", "coded sp", "coded ap"),
                          (t, f0, sp, ap, ct, cf0, csp, cap), full + coded):
        assert torch.equal(a, b), name
    assert (f0 > 0).sum() > 20 and np.isfinite(pc.to_np(csp)).all()
