"""Voice transformation (world_b200_transform_batch / world_b200_transform_host) on the single-thread host emulation of
the kernel sources (CPU): every output row equals the library's stepwise chain bit for bit."""
import pytest

import transform_common as tc


@pytest.mark.parametrize("fs,fft,method,nbit", [(16000, 1024, "harvest", 16), (22050, 1024, "dio", 24),
                                                (48000, 2048, "harvest", 0), (16000, 1024, "dio", 0)])
def test_emu_transform_equals_stepwise(emu, fs, fft, method, nbit):
    tc.check_stepwise(emu, fs, fft, method, nbit, seconds=0.4)


def test_emu_transform_relaid_pass(emu):
    tc.check_relaid_pass(emu)


def test_emu_transform_null_factors(emu):
    tc.check_null_factors(emu)


@pytest.mark.parametrize("method", ["harvest", "dio"])
def test_emu_transform_per_utterance_options(emu, method):
    tc.check_per_utterance_options(emu, method)


def test_emu_transform_small_budget(emu):
    tc.check_small_budget(emu, seconds=2.0)


def test_emu_transform_host_equals_device(emu):
    tc.check_host_equals_device(emu)


def test_emu_transform_invalid(emu):
    tc.check_invalid(emu)


def test_emu_transform_time_scale_vs_reference(emu, ref, golden):
    tc.check_time_scale_vs_reference(emu, ref, golden)
