"""The per-utterance CheapTrick / D4C overloads of include/world_b200.hpp (tests/cpp/spectral_options_overload.cpp): they
compile and link against the library; on the GPU every row equals the single-utterance CheapTrick() / D4C() at that
utterance's own option."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
CUDA_INC = "/usr/local/cuda/include"
CUDA_LIB = "/usr/local/cuda/lib64"


def build_program(out):
    from world_b200 import api
    libdir = os.path.dirname(api.DEFAULT_LIB)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", INC, "-I", CUDA_INC,
                           os.path.join(ROOT, "tests", "cpp", "spectral_options_overload.cpp"), "-o", str(out),
                           "-L", libdir, "-lworld_b200", "-L", CUDA_LIB, "-lcudart",
                           f"-Wl,-rpath,{libdir}", f"-Wl,-rpath,{CUDA_LIB}"])
    return str(out)


def test_cpp_spectral_options_overload_compiles_and_fails_loudly_without_gpu(tmp_path):
    exe = build_program(tmp_path / "spectral_options_overload")
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0
    assert "no CPU path" in r.stderr


@pytest.mark.gpu
def test_gpu_cpp_spectral_options_overload_equals_single_utterance_api(tmp_path):
    exe = build_program(tmp_path / "spectral_options_overload")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
