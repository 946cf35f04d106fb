"""harvest_contour_kernel's warp reductions on candidate maps built to reach their edge cases: SelectBestF0 in ExtendF0
(one warp per section, lanes over the candidate slots, the warp keeping the smallest error and the LAST slot among
equal errors) and SearchScore in MergeF0Sub (one warp per frame of the overlap, the warp maximum from +0.0 with the
reference's strict `<`, the terms summed in ascending frame order in rounds of 128 frames).  A slot j sits in lane
j % 32, so the pairs below put equal candidates in one lane, in two lanes either way round, and in lanes 31 and 0 of
consecutive words.  Everything is compared bit for bit against the reference's own functions through
f0_tail_common; the branch each map was built for is asserted on the reference's output."""
import f0_tail_common as ft

F = 100.0                 # a section at exactly 100 Hz: |100 - 96| / 100 and |100 - 104| / 100 are the same double
SEC, GAP = 50, 300        # a section's frames, and the distance between sections of one map
PAIRS = [(0, 1), (1, 0), (3, 35), (35, 3), (33, 40), (40, 33), (31, 32), (32, 31), (100, 4), (4, 100), (139, 2)]
RANGES = {105: ft.R_DEFAULT, 140: ft.R_WIDE, 84: (100.0, 600.0), 7: ft.R_DEFAULT}   # nc * 7 -> a range that has it


def _sections(nc7, n):
    m = ft.empty(GAP * n + 200, nc7 // 7, RANGES[nc7])
    return m, [150 + GAP * k for k in range(n)]


def _section(m, a):
    m.cand[a:a + SEC, 0], m.score[a:a + SEC, 0] = F, 5.0


def tie_map(nc7):
    """After each section, 20 frames with 96 Hz in slot a and 104 Hz in slot b (and before it the same, mirrored):
    both are 0.04 from the section's last value, so ExtendF0 goes on with the one in the higher slot, both ways."""
    pairs = [(a, b) for a, b in PAIRS if a < nc7 and b < nc7]
    m, starts = _sections(nc7, len(pairs))
    m.name = f"ties({nc7} slots)"
    for (a, b), p in zip(pairs, starts):
        _section(m, p)
        m.cand[p + SEC:p + SEC + 20, a], m.cand[p + SEC:p + SEC + 20, b] = 96.0, 104.0
        m.cand[p - 20:p, b], m.cand[p - 20:p, a] = 96.0, 104.0
    return m, [(a, b, p) for (a, b), p in zip(pairs, starts)]


def allowed_map(nc7):
    """Errors of exactly allowed_range (0.18): 118 Hz alone is taken; 82 Hz in slot a against 118 Hz in slot b is a tie
    at the bound, the higher slot wins; 118 Hz raised by one part in 2^40 is out of range and the extension misses."""
    a, b = 1, min(nc7 - 1, 40)
    m, starts = _sections(nc7, 3)
    m.name = f"allowed({nc7} slots)"
    for p in starts:
        _section(m, p)
    p0, p1, p2 = starts
    m.cand[p0 + SEC:p0 + SEC + 10, b] = 118.0
    m.cand[p1 + SEC:p1 + SEC + 10, a], m.cand[p1 + SEC:p1 + SEC + 10, b] = 82.0, 118.0
    m.cand[p2 + SEC:p2 + SEC + 10, b] = 118.0 * (1 + 2.0 ** -40)
    return m, starts


def merge_map(a_tail, dup_slots, dup_scores, nc=15):
    """Section A (100 Hz, slot 0, frames 50 .. 300 at score 5) runs on at score a_tail to frame 401, section B (150 Hz,
    slot 1, frames 310 .. 500 at score 5) reaches back at score 0 to frame 209: an overlap of more than 190 frames, two
    rounds of terms.  A's values of frames 220 .. 260 appear again in dup_slots with dup_scores: SearchScore takes the
    largest score of the slots that hold the value, slot 0's 5 included."""
    m = ft.empty(700, nc, name=f"merge({a_tail}, {dup_slots}, {dup_scores})")
    ft.put(m, 0, ft.FA, 50, 300, 5.0); ft.put(m, 0, ft.FA, 301, 401, a_tail)
    ft.put(m, 1, ft.FB, 209, 309, 0.0); ft.put(m, 1, ft.FB, 310, 500, 5.0)
    for s, sc in zip(dup_slots, dup_scores):
        m.cand[220:261, s], m.score[220:261, s] = m.cand[220:261, 0], sc
    return m


def check_select(world, tail):
    maps, cases = [], []
    for nc7 in (105, 140, 84, 7):
        mt, ties = tie_map(nc7)
        ma, allowed = allowed_map(nc7)
        maps += [mt, ma]
        cases += [("ties", ties), ("allowed", allowed)]
    rep = ft.Report()
    res = ft.check_batch(world, tail, maps, rep=rep, what="select")
    for m, (kind, case), (steps, _) in zip(maps, cases, res):
        s3 = steps[3]
        if kind == "ties":
            for a, b, p in case:
                hi = 104.0 if b > a else 96.0
                assert s3[p + SEC] == hi and s3[p - 1] == (96.0 if b > a else 104.0), f"{m.name}: slots {a}, {b}"
        else:
            p0, p1, p2 = case
            assert s3[p0 + SEC] == 118.0, f"{m.name}: an error of exactly 0.18 is in range"
            assert s3[p1 + SEC] == 118.0, f"{m.name}: 82 and 118 tie at the bound, the higher slot wins"
            assert s3[p2 + SEC] == 0.0, f"{m.name}: just above 0.18 is out of range"
    # more sections than the CTA has warps, each with its own tie
    assert sum(len(c) for k, c in cases if k == "ties") > 8
    return rep


def check_merge(world, tail):
    maps = [merge_map(0.0, (), ()), merge_map(1.0, (), ()), merge_map(0.0, (37, 70), (6.0, 9.0)),
            merge_map(0.0, (70, 37), (6.0, 9.0)), merge_map(0.0, (31, 32, 104), (2.0, 7.0, 6.5)),
            merge_map(0.0, (40, 8), (3.0, 1.0))]
    rep = ft.Report()
    res = ft.check_batch(world, tail, maps, rep=rep, what="merge")
    on_a = [steps[3][250] == ft.track(ft.FA, 250, 0) for steps, _ in res]
    # A scores 5 up to frame 300 and B 5 from frame 310 on, which is the larger sum: B from st2.  A's run-on at score 1
    # adds about 100 to A's side, duplicates scoring 9 or 7 add 41 * 4 or 41 * 2; those scoring below 5 add nothing
    assert on_a == [False, True, True, True, True, False], on_a
    assert all(steps[3][450] == ft.track(ft.FB, 450, 1) for steps, _ in res)
    return rep
