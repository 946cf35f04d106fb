"""Per-utterance DIO options over two ranks (gloo, host emulation): each rank passes the options of its own
utterance shard, and the gathered f0 rows are bit-identical to one process analysing the whole batch."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FS, N = 16000, 6400
LENS = [6400, 5000, 6400, 4200, 6000]
RANGES = [(40.0, 1100.0, 2.0, 0.1), (71.0, 800.0, 3.0, 0.1), (100.0, 600.0, 2.0, 0.2), (50.0, 300.0, 2.0, 0.1),
          (71.0, 800.0, 3.0, 0.05)]

WORKER = r'''
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import numpy as np, torch, torch.distributed as dist
from world_b200.api import World
from world_b200.shard import shard_ranges, all_gather_rows
from synth import synth_batch
import dio_ranges_common as fr
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
fs, n, lens, ranges = {fs}, {n}, {lens!r}, {ranges!r}
x = synth_batch(range(1, 6), fs, n).numpy()
w = World(lib_path=os.path.join({root!r}, "tests", "emu", "libworld_b200_emu.so"), array_module="numpy")
frames = [w.frames(fs, l) for l in lens]
L = max(frames)
b, e = shard_ranges(frames, world)[rank]
f0 = np.zeros((e - b, L))
if e > b:
    t, f, fl = w.dio(np.ascontiguousarray(x[b:e]), fs, fr.options(ranges[b:e]), x_lengths=lens[b:e])
    w.synchronize()
    f0[:, :f.shape[1]] = f
counts = [r[1] - r[0] for r in shard_ranges(frames, world)]
g = all_gather_rows(dist, torch.from_numpy(f0), counts).numpy()
if rank == 0:
    np.save({out!r}, g)
dist.destroy_process_group()
'''


def test_two_rank_per_utterance_dio_options_equal_single_process(emu, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dio_ranges_common as fr
    from synth import synth_batch
    out = str(tmp_path / "f0.npy")
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, out=out, fs=FS, n=N, lens=LENS, ranges=RANGES))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                           "--master-addr", "127.0.0.1", "--master-port", "29542", str(script)], env=env,
                          timeout=600)
    got = np.load(out)
    x = synth_batch(range(1, 6), FS, N).numpy()
    t, f0, fl = emu.dio(x, FS, fr.options(RANGES), x_lengths=LENS)
    emu.synchronize()
    assert got.shape == f0.shape
    assert np.array_equal(got, f0)
