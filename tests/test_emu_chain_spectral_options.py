"""The full-row analysis chains with one CheapTrick / D4C option per utterance, on the single-thread host emulation of
the kernel sources (CPU): against each speaker's group run alone, the padded layout, equal options, the reference,
lane slices and host chunks, the EINVAL rules, and two ranks gathered with gloo."""
import os
import subprocess
import sys

import numpy as np
import pytest

import chain_spectral_options_common as cs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("method", ["harvest", "dio"])
@pytest.mark.parametrize("f0_options", [True, False])
def test_emu_chain_spectral_options_groups(emu, method, f0_options):
    cs.check_groups(emu, 16000, 3200, 6, method=method, f0_options=f0_options)


def test_emu_chain_spectral_options_layout(emu):
    cs.check_layout(emu, 16000, 3200)


@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_emu_chain_spectral_options_identity(emu, method):
    cs.check_identity(emu, 16000, 3200, method=method)


@pytest.mark.parametrize("fs,n", [(16000, 4000), (22050, 4410)])
@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_emu_chain_spectral_options_vs_reference(emu, ref, fs, n, method):
    cs.check_vs_ref(emu, ref, fs, n, method=method)


def test_emu_chain_spectral_options_slices_and_chunks(emu):
    cs.check_slices_and_chunks(emu, 16000, 3200, 7)


def test_emu_chain_spectral_options_invalid(emu):
    cs.check_invalid(emu)


WORKER = r'''
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import numpy as np, torch, torch.distributed as dist
from world_b200.api import World
from world_b200.shard import all_gather_rows
import chain_spectral_options_common as cs
dist.init_process_group("gloo")
rank = dist.get_rank()
w = World(lib_path=os.path.join({root!r}, "tests", "emu", "libworld_b200_emu.so"), array_module="numpy")
c = cs.Case(w, {fs}, {n}, {n_utts})
L, W = max(c.frames), c.width
b, e = {shards!r}[rank]
outs = [np.zeros((e - b, L)), np.zeros((e - b, L)), np.zeros((e - b, L, W)), np.zeros((e - b, L, W))]
w.analyze_batch(np.ascontiguousarray(c.x[b:e]), c.fs, c.ao, x_lengths=c.lens[b:e], time_axis=outs[0], f0=outs[1],
                spectrogram=outs[2], aperiodicity=outs[3], **{{k: v[b:e] for k, v in c.kw.items()}})
w.synchronize()
g = [all_gather_rows(dist, torch.from_numpy(a), [e - b for b, e in {shards!r}]).numpy() for a in outs]
if rank == 0:
    np.savez({out!r}, t=g[0], f0=g[1], sp=g[2], ap=g[3])
dist.destroy_process_group()
'''


def test_two_rank_full_rows_gather_equals_single_process(emu, tmp_path):
    """Two ranks whose shards' largest sizes differ (2048 and 1024 at 16 kHz) write rows of one common row_stride, the
    largest of the whole batch; the gathered arrays equal one process analysing the whole batch, pads included."""
    fs, n, n_utts, shards = 16000, 4000, 4, [(0, 2), (2, 4)]
    c = cs.Case(emu, fs, n, n_utts)
    assert len({max(c.sizes[b:e]) for b, e in shards}) == 2
    out = str(tmp_path / "full.npz")
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, out=out, fs=fs, n=n, n_utts=n_utts, shards=shards))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                           "--master-addr", "127.0.0.1", "--master-port", "29547", str(script)], env=env,
                          timeout=600)
    got = np.load(out)
    want = c.run(emu)
    for name, w in zip(("t", "f0", "sp", "ap"), want):
        assert got[name].shape == w.shape, name
        assert np.array_equal(got[name], w), name
    assert (want[1] > 0).sum() > 20
