"""The F0 decision stages (Harvest after candidate refinement, DIO's contour) on constructed candidate maps against
the reference's own functions, on the CUDA library (-m gpu).  Beyond what the emulation runs, this is where
hv_boundaries splits its scan over the block's threads, where harvest_remove_kernel's warp arg-max breaks score ties
across lanes, and where sections are extended and filtered by one thread each."""
import pytest

import f0_tail_common as ft
from f0_tail_common import tail  # noqa: F401  (fixture)


def _report(name, rep):
    print(f"\n{name}: {rep.maps} maps, {rep.frames} frames, {rep.sections} sections ({rep.merged} merged away); "
          f"smoothed f0 worst {rep.smooth_worst:.2e} of the peak (bound {ft.SMOOTH_BOUND:.2e})")


@pytest.mark.gpu
def test_gpu_f0_tail_wrapper_pin(gpu_world, ref, tail, golden):
    ft.check_wrapper_pin(gpu_world, ref, tail, golden)


@pytest.mark.gpu
@pytest.mark.parametrize("check", [ft.check_merge, ft.check_extend, ft.check_ties_and_counts, ft.check_frame_periods,
                                   ft.check_ragged_batch, ft.check_dense], ids=lambda f: f.__name__[6:])
def test_gpu_f0_tail_directed(gpu_world, tail, check):
    _report(check.__name__, check(gpu_world, tail))


@pytest.mark.gpu
def test_gpu_f0_tail_random(gpu_world, tail):
    rep = ft.check_random(gpu_world, tail, 600, seed=2, per_call=100)
    _report("random", rep)
    assert rep.maps == 600 and rep.sections > 6000 and rep.merged > 3000, rep


@pytest.mark.gpu
def test_gpu_f0_tail_load_errors(gpu_world, tail):
    ft.check_load_errors(gpu_world, tail)


@pytest.mark.gpu
def test_gpu_f0_tail_dio(gpu_world, tail):
    compared, voiced = ft.check_dio(gpu_world, tail)
    print(f"\ndio: {compared} frames compared bit for bit, {voiced} voiced")
