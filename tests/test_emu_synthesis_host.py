"""Synthesis from coded rows to 16-bit PCM (world_b200_synthesis_coded_batch_pcm16) and the pipelined host call
(world_b200_synthesis_coded_host) on the single-thread host emulation of the kernel sources (CPU)."""
import pytest

import synthesis_host_common as sh


@pytest.mark.parametrize("fs,fp,dims", [(16000, 5.0, 60), (16000, 2.5, 40), (22050, 2.5, 60), (48000, 5.0, 40)])
def test_emu_synthesis_pcm16_equals_quantised(emu, fs, fp, dims, tmp_path):
    sh.check_pcm_equals_quantised(emu, fs, fp, dims, tmp_path)


def test_emu_synthesis_pcm16_clips(emu):
    sh.check_pcm_clips(emu)


def test_emu_synthesis_host_equals_device(emu):
    sh.check_host_equals_device(emu)


def test_emu_synthesis_host_pipeline_chunks(emu, capfd, monkeypatch):
    sh.check_pipeline_chunks(emu, capfd, monkeypatch)


def test_emu_synthesis_host_high_f0(emu):
    sh.check_host_high_f0(emu)


def test_emu_synthesis_pcm16_vs_reference(emu, ref, golden):
    print(f"worst {sh.check_vs_reference(emu, ref, golden)} LSB")


def test_emu_synthesis_host_no_bands(emu):
    sh.check_no_bands(emu)


def test_emu_synthesis_host_invalid(emu):
    sh.check_invalid(emu)
