"""DIO at every rate, speed and floor on voices that start or end abruptly, on the CUDA library: against the reference,
against its own call on the utterance alone, and with poisoned scratch."""
import pytest

import dio_rate_edges_common as de

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ceil", de.CEILS)
@pytest.mark.parametrize("speed", de.SPEEDS)
@pytest.mark.parametrize("fs", de.RATES)
def test_gpu_dio_rate_edges_vs_reference(gpu_world, ref, fs, speed, ceil):
    de.check_vs_ref(gpu_world, ref, fs, speed, ceil)


@pytest.mark.parametrize("fs,speed", [(48000, 1), (44100, 1), (48000, 2), (32000, 1), (22050, 1)])
def test_gpu_dio_rate_edges_lone_call(gpu_world, fs, speed):
    de.check_lone(gpu_world, fs, speed, floors=(40.0, 45.0, 50.0, 55.0))


@pytest.mark.parametrize("fs", [48000, 16000])
def test_gpu_dio_rate_edges_poisoned_scratch(gpu_world, fs):
    de.check_poison(gpu_world, fs)
