"""F0 scaling and formant shift (world_b200_modify_batch, world_b200_synthesis_coded_*_modified) on the single-thread
host emulation of the kernel sources (CPU).  The emulation evaluates log / exp with the host's libm, as the restatement
does, so its envelopes are held to the reference bit for bit."""
import os

import pytest

import modify_common as mc


def test_emu_modify_golden_vs_reference(emu, ref, golden):
    mc.check_golden(emu, ref, golden, exact=True)


@pytest.mark.parametrize("fs,fft", [(16000, 512), (16000, 1024), (22050, 1024), (48000, 2048)])
def test_emu_modify_analysed_vs_reference(emu, ref, fs, fft):
    mc.check_analysed(emu, ref, fs, fft, exact=True)


def test_emu_modify_identity_and_bounds(emu):
    mc.check_identity_and_bounds(emu)


def test_emu_modify_fused_equals_stepwise(emu):
    mc.check_fused_equals_stepwise(emu)


def test_emu_modify_small_budget(emu):
    mc.check_small_budget(emu)


def test_emu_modify_scaled_high_f0(emu):
    mc.check_scaled_high_f0(emu)


def test_emu_modify_host_equals_device(emu):
    mc.check_host_equals_device(emu)


def test_emu_modify_invalid(emu):
    mc.check_invalid(emu)


def test_ref_demo_builds_and_runs(golden, tmp_path):
    """The reference's demo (test/test.cpp), compiled unchanged, runs on the fixture and writes its modified synthesis."""
    if not os.path.exists(mc.REF_DEMO):
        pytest.skip("oracle/_ref/ref_demo missing: build() found no reference sources")
    y = mc.run_ref_demo(golden, str(tmp_path), 1.5, 0.85)
    assert len(y) > 10000 and abs(y).max() > 1000
