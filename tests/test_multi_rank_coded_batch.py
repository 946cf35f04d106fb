"""The coded device chain over two ranks (gloo, host emulation): each rank analyses its utterance shard from int16 PCM
with analyze_coded_batch, the coded shards are gathered with world_b200.shard.all_gather_rows, and every gathered
array is bit-identical to one process analysing the whole batch."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FS, N, DIMS = 16000, 6400, 24
LENS = [6400, 5000, 6400, 4200, 6000]

WORKER = r'''
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import numpy as np, torch, torch.distributed as dist
from world_b200.api import World, F0_HARVEST
from world_b200.shard import shard_ranges, all_gather_rows
from synth import synth_batch
import coded_batch_common as cb
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
fs, n, lens, dims = {fs}, {n}, {lens!r}, {dims}
pcm, _ = cb.pcm_rows(0.5 * synth_batch(range(1, 6), fs, n).numpy(), 16)
w = World(lib_path=os.path.join({root!r}, "tests", "emu", "libworld_b200_emu.so"), array_module="numpy")
ao = w.analysis_option(fs, F0_HARVEST)
frames = [w.frames(fs, l) for l in lens]
L, n_ap = max(frames), w.number_of_aperiodicities(fs)
ranges = shard_ranges(frames, world)
b, e = ranges[rank]
outs = [np.zeros((e - b, L)), np.zeros((e - b, L)), np.zeros((e - b, L, dims)), np.zeros((e - b, L, n_ap))]
if e > b:
    w.analyze_coded_batch(np.ascontiguousarray(pcm[b:e]), 16, fs, ao, dims, x_lengths=lens[b:e], time_axis=outs[0],
                          f0=outs[1], coded_sp=outs[2], coded_ap=outs[3])
    w.synchronize()
counts = [r[1] - r[0] for r in ranges]
g = [all_gather_rows(dist, torch.from_numpy(a), counts).numpy() for a in outs]
if rank == 0:
    np.savez({out!r}, t=g[0], f0=g[1], csp=g[2], cap=g[3])
dist.destroy_process_group()
'''


def test_two_rank_coded_gather_equals_single_process(emu, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import coded_batch_common as cb
    from synth import synth_batch
    from world_b200.api import F0_HARVEST
    out = str(tmp_path / "coded.npz")
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, out=out, fs=FS, n=N, lens=LENS, dims=DIMS))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                           "--master-addr", "127.0.0.1", "--master-port", "29543", str(script)], env=env,
                          timeout=600)
    got = np.load(out)
    pcm, _ = cb.pcm_rows(0.5 * synth_batch(range(1, 6), FS, N).numpy(), 16)
    t, f0, csp, cap, fl = emu.analyze_coded_batch(pcm, 16, FS, emu.analysis_option(FS, F0_HARVEST), DIMS,
                                                  x_lengths=LENS)
    emu.synchronize()
    for name, want in (("t", t), ("f0", f0), ("csp", csp), ("cap", cap)):
        assert got[name].shape == want.shape, name
        assert np.array_equal(got[name], want), name
    assert (f0 > 0).sum() > 50
