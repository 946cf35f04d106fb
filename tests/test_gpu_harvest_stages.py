"""Harvest stage by stage against extended-precision restatements, on the CUDA library (-m gpu): the tensor-core
filter bank, the event trains and the DMMA refinement as the GPU sums them.  Every third 1 ms frame of the
refinement is restated."""
import pytest

import harvest_stages_common as hs

R_EVEN, R_ODD = (71.0, 800.0), (40.0, 1100.0)   # 152 and 203 bands: the odd count leaves one band unpaired
SPEECHY = ["speech", "tone", "impulses", "dc", "clipped"]


def _report(name, out):
    f, s = out["refined"]
    print(f"\n{name}: decimated {out['decimated']:.2e} of the peak; raw worst {out['raw'].worst:.2e} "
          f"(bound {out['raw'].worst_bound:.2e}, {out['raw'].compared} compared, {out['raw'].excluded} excluded); "
          f"base {out['base']} bit-equal; refined f0 {f.worst:.2e} (bound {f.worst_bound:.2e}), score {s.worst:.2e} "
          f"(bound {s.worst_bound:.2e}), {f.compared} compared, {f.excluded} excluded")


@pytest.mark.gpu
@pytest.mark.parametrize("name,fs,lens,ranges,env", [
    # decimated lengths 4096 (four FIR tiles), 4095, 4097 and 700 (shorter than the 875-tap band of the 40 Hz
    # floor); two range groups, one of them with an odd band count
    ("chain_16k", 16000, [8192, 8190, 8194, 1400, 5000], [R_EVEN, R_ODD], None),
    ("chain_12k", 12000, [6000, 4500], [R_EVEN], None),
    ("chain_48k", 48000, [12288, 9000], [R_ODD, R_EVEN], None),
    ("per_frame_22k", 22050, [8000, 6615], [R_EVEN], None),
    ("per_frame_44k", 44100, [13000, 11025], [R_ODD], None),
    ("streaming_16k", 16000, [8194, 6000], [R_EVEN], {"WB_SWEEP_STREAMING": "1"}),
    ("ripple_8k", 8000, [4096, 3000], [R_EVEN, R_ODD], None),
    ("ripple_11k", 11025, [4000, 5513], [R_EVEN], None),
    ("no_chain_16k", 16000, [8192, 5000], [R_ODD], {"WB_NO_REFINE_CHAIN": "1"}),
])
def test_gpu_harvest_stages(gpu_world, ref, name, fs, lens, ranges, env):
    kinds = [SPEECHY[u % len(SPEECHY)] for u in range(len(lens))]
    _report(name, hs.run_case(gpu_world, ref, fs, kinds, lens, ranges, env=env, frame_step=3))


@pytest.mark.gpu
def test_gpu_harvest_stages_redo_list(gpu_world, ref):
    """the loud tone of check_event_dense_and_degenerate_bands with rings of 64 events: bands redone"""
    _report("redo_list", hs.run_case(gpu_world, ref, 22050, ["tone"], [19000], [(71.0, 800.0)],
                                     env={"WB_EDGE_CAP_MIN": "64"}, frame_step=3))


@pytest.mark.gpu
def test_gpu_harvest_stages_last_chunk(gpu_world, ref):
    _report("last_chunk", hs.check_last_chunk(gpu_world, ref, frame_step=3))
