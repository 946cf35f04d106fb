"""Harvest stage by stage against extended-precision restatements, on the single-thread host emulation of the kernel
sources (CPU).  Short signals and every ninth 1 ms frame of the refinement keep this file near a minute."""
import pytest

import harvest_stages_common as hs

R_EVEN, R_ODD = (71.0, 800.0), (40.0, 1100.0)   # 152 and 203 bands: the odd count leaves one band unpaired


@pytest.mark.parametrize("name,fs,kinds,lens,ranges,env", [
    # decimated lengths 2048 (two FIR tiles), 2047, 2049 and 700 (shorter than the 875-tap band of the 40 Hz floor),
    # two range groups in one call
    ("split_tiles_groups", 16000, ["speech", "tone", "impulses", "dc"], [4096, 4094, 4098, 1400], [R_EVEN, R_ODD], None),
    ("per_frame_22k", 22050, ["clipped", "speech"], [5000, 4410], [R_EVEN], None),
    ("streaming_16k", 16000, ["speech", "dc"], [4098, 3000], [R_EVEN], {"WB_SWEEP_STREAMING": "1"}),
    ("ripple_8k", 8000, ["speech", "impulses"], [2049, 2400], [R_EVEN, R_ODD], None),
    ("redo_list", 22050, ["tone"], [6000], [(71.0, 800.0)], {"WB_EDGE_CAP_MIN": "64"}),
    ("no_chain_16k", 16000, ["speech", "clipped"], [4096, 3500], [R_ODD], {"WB_NO_REFINE_CHAIN": "1"}),
])
def test_emu_harvest_stages(emu, ref, name, fs, kinds, lens, ranges, env):
    hs.run_case(emu, ref, fs, kinds, lens, ranges, env=env, frame_step=9)


def test_emu_harvest_stages_last_chunk(emu, ref):
    hs.check_last_chunk(emu, ref, frame_step=9)
