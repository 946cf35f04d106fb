"""harvest_contour_kernel's SelectBestF0 and SearchScore reductions on constructed maps, on the CUDA library (-m gpu):
here the candidate slots are spread over the 32 lanes of a warp and sections over the CTA's four warps."""
import pytest

import contour_reductions_common as cr
from f0_tail_common import tail  # noqa: F401  (fixture)


@pytest.mark.gpu
def test_gpu_contour_select_best(gpu_world, tail):
    cr.check_select(gpu_world, tail)


@pytest.mark.gpu
def test_gpu_contour_search_score(gpu_world, tail):
    cr.check_merge(gpu_world, tail)
