import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


# GPU tests of the newest code (DIO's ripple path, event rings, drop-in programs) run after the others: with
# `pytest -x` an early surprise must not hide the rest.
_RUN_LAST = ("golden_dio", "dio_path", "dio_decimated", "edge_cases", "long_48k", "legacy_api_and_analyze_host",
             "analyze_coded_host", "host_pipeline_chunking", "event_dense", "zero_tail_f0", "mirroring_ripple",
             "reference_examples", "cpp_batched")


def pytest_collection_modifyitems(config, items):
    items.sort(key=lambda it: 1 if ("gpu" in it.keywords and any(k in it.name for k in _RUN_LAST)) else 0)
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference, compiled into oracle/_ref by build() where its sources are present."""
    from refworld import RefWorld, REF_LIB
    if not os.path.exists(REF_LIB):
        pytest.skip("oracle/_ref/libworld_ref.so missing: build() found no reference sources")
    return RefWorld(REF_LIB)


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "vaiueo2d.npz"))


@pytest.fixture(scope="session")
def emu():
    """Single-thread host emulation of the kernel sources (logic check without a GPU)."""
    from world_b200.api import World
    path = os.path.join(ROOT, "tests", "emu", "libworld_b200_emu.so")
    subprocess.check_call([os.path.join(ROOT, "tests", "emu", "build.sh")], stdout=subprocess.DEVNULL)
    # WB_EMU_LIB: an instrumented build of the same sources (e.g. -fsanitize=address, see tests/emu/README)
    return World(lib_path=os.environ.get("WB_EMU_LIB", path), array_module="numpy")


@pytest.fixture(scope="session")
def gpu_world():
    import torch
    from world_b200.api import World
    torch.cuda.set_device(0)
    return World(device=0)
