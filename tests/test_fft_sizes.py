"""CheapTrick, D4C, the codec and Synthesis at every FFT size they accept, against the reference (fft_sizes_common):
a reduced grid on the host emulation (CPU suite) and the full grid on the CUDA library (-m gpu)."""
import pytest

import fft_sizes_common as fz


# ---------------------------------------------------------------- the emulation (CPU suite) ...
def test_emu_cheaptrick_sizing_helpers(emu, ref):
    print(f"{fz.check_sizing_helpers(emu, ref)} f0_floor values")


@pytest.mark.parametrize("fs,sizes", [(8000, [16, 64, 128]), (22050, [32, 256, 8192]), (48000, [512, 4096])])
def test_emu_cheaptrick_sizes(emu, ref, fs, sizes):
    print(fz.table(fz.check_cheaptrick(emu, ref, fs, sizes), "CheapTrick"))


@pytest.mark.parametrize("fs,fft", [(8000, 32), (44100, 256)])
def test_emu_cheaptrick_below_the_500_hz_window(emu, ref, fs, fft):
    print(f"fs {fs} fft {fft}: worst {fz.check_cheaptrick_edomain(emu, ref, fs, fft):.1e}")


@pytest.mark.parametrize("fs,sizes", [(16000, [4, 64, 3001]), (44100, [16, 1000, 8192])])
def test_emu_d4c_sizes(emu, ref, fs, sizes):
    print(fz.table(fz.check_d4c(emu, ref, fs, sizes), "D4C"))


def test_emu_d4c_tiny_sizes_refused(emu):
    fz.check_d4c_tiny_sizes_refused(emu)


@pytest.mark.parametrize("fs", [8000, 16000, 44100])
def test_emu_codec_sizes(emu, ref, fs):
    print(fz.table(fz.check_codec(emu, ref, fs, fz.POW2, fz.POW2 + [1000, 3001]), "codec"))


@pytest.mark.parametrize("fs,sizes", [(8000, [16, 32, 256]), (22050, [64, 128, 2048]), (48000, [16, 128, 4096])])
def test_emu_synthesis_sizes(emu, ref, fs, sizes):
    print(fz.table(fz.check_synthesis(emu, ref, fs, sizes), "Synthesis"))


@pytest.mark.parametrize("fs,f0_floor,method", fz.CHAIN_CASES[:1])
def test_emu_chain_at_another_f0_floor(emu, ref, fs, f0_floor, method):
    fft, worst = fz.check_chain_option(emu, ref, fs, f0_floor, method)
    print(f"fs {fs} f0_floor {f0_floor} (fft {fft}): worst {worst:.1e}")


# ---------------------------------------------------------------- ... and the CUDA library
@pytest.mark.gpu
def test_gpu_cheaptrick_sizing_helpers(gpu_world, ref):
    print(f"{fz.check_sizing_helpers(gpu_world, ref)} f0_floor values")


@pytest.mark.gpu
@pytest.mark.parametrize("fs", fz.CT_RATES)
def test_gpu_cheaptrick_sizes(gpu_world, ref, fs):
    print(fz.table(fz.check_cheaptrick(gpu_world, ref, fs, fz.POW2), "CheapTrick"))


@pytest.mark.gpu
@pytest.mark.parametrize("fs", fz.CT_RATES)
def test_gpu_cheaptrick_below_the_500_hz_window(gpu_world, ref, fs):
    fft = max(s for s in fz.POW2 if not fz.ct_defined(fs, s))
    print(f"fs {fs} fft {fft}: worst {fz.check_cheaptrick_edomain(gpu_world, ref, fs, fft):.1e}")


@pytest.mark.gpu
@pytest.mark.parametrize("fs", fz.D4C_RATES)
def test_gpu_d4c_sizes(gpu_world, ref, fs):
    print(fz.table(fz.check_d4c(gpu_world, ref, fs, fz.D4C_SIZES), "D4C"))


@pytest.mark.gpu
def test_gpu_d4c_tiny_sizes_refused(gpu_world):
    fz.check_d4c_tiny_sizes_refused(gpu_world)


@pytest.mark.gpu
@pytest.mark.parametrize("fs", fz.CT_RATES)
def test_gpu_codec_sizes(gpu_world, ref, fs):
    print(fz.table(fz.check_codec(gpu_world, ref, fs, fz.POW2, fz.POW2 + [1000, 3001]), "codec"))


@pytest.mark.gpu
@pytest.mark.parametrize("fs", fz.SYNTHESIS_RATES)
def test_gpu_synthesis_sizes(gpu_world, ref, fs):
    print(fz.table(fz.check_synthesis(gpu_world, ref, fs, fz.SYNTHESIS_SIZES), "Synthesis"))


@pytest.mark.gpu
@pytest.mark.parametrize("fs,f0_floor,method", fz.CHAIN_CASES)
def test_gpu_chain_at_another_f0_floor(gpu_world, ref, fs, f0_floor, method):
    fft, worst = fz.check_chain_option(gpu_world, ref, fs, f0_floor, method)
    print(f"fs {fs} f0_floor {f0_floor} (fft {fft}): worst {worst:.1e}")
