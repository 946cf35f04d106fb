"""harvest_contour_kernel's SelectBestF0 and SearchScore reductions on constructed maps, on the single-thread host
emulation of the kernel sources (CPU)."""
import contour_reductions_common as cr
from f0_tail_common import tail  # noqa: F401  (fixture)


def test_emu_contour_select_best(emu, tail):
    cr.check_select(emu, tail)


def test_emu_contour_search_score(emu, tail):
    cr.check_merge(emu, tail)
