"""The F0 decision stages on candidate maps the test constructs: Harvest's RemoveUnreliableCandidates, FixF0Contour
and SmoothF0Contour (harvest_remove_kernel, harvest_contour_kernel, harvest_smooth_kernel) and DIO's GetBestF0Contour
and FixF0Contour (dio_contour_kernel), against the reference's own functions (oracle/ref_f0_tail.cpp compiles them
into oracle/_ref/libworld_ref_tail.so).  The library is driven through its public calls: WB_LOAD_REFINED /
WB_LOAD_DIO_CAND replace the candidate rows in front of those kernels, which then run as harvest_run / dio_run
launch them; WB_DUMP_CLEANED / WB_DUMP_CONTOUR capture what is between them.  The stages are selections, so everything
is compared bit for bit except the smoothing filter (bound below).  Each directed case states, on the reference's
output, which branch it was built to take.  The same checks run on the host emulation and on the CUDA library."""
import ctypes as C
import math
import os
import struct
import tempfile
from dataclasses import dataclass

import numpy as np
import pytest

import harvest_stages_common as hs
import test_parity_common as pc
from refworld import REF_LIB
from world_b200.api import WorldError

TAIL_LIB = os.path.join(os.path.dirname(REF_LIB), "libworld_ref_tail.so")
_P = C.c_void_p
FS = 4000                      # four samples per 1 ms frame, no decimation: the stages in front cost next to nothing
R_DEFAULT, R_WIDE = (71.0, 800.0), (40.0, 1100.0)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same_bits(a, b):
    return np.array_equal(bits(a), bits(b))


class RefTail:
    def __init__(self):
        if not os.path.exists(TAIL_LIB):
            pytest.skip("oracle/_ref/libworld_ref_tail.so missing: build() found no reference sources")
        self.lib = C.CDLL(TAIL_LIB, mode=os.RTLD_LOCAL | os.RTLD_NOW)
        self.lib.RefHarvestTail.restype = None
        self.lib.RefHarvestTail.argtypes = [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P]
        self.lib.RefDioContour.restype = None
        self.lib.RefDioContour.argtypes = [C.c_double, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.c_double,
                                           C.c_double, _P, _P]

    def harvest_tail(self, cand, score, n_cand):
        """cand, score: [L][max_cand] -> cleaned cand, cleaned score, steps[5][L] (base, FixStep1..4), f0 at 1 ms"""
        cand, score = np.ascontiguousarray(cand), np.ascontiguousarray(score)
        L, mc = cand.shape
        cc, cs = np.zeros_like(cand), np.zeros_like(score)
        steps, contour, f0 = np.zeros((5, L)), np.zeros(L), np.zeros(L)
        self.lib.RefHarvestTail(cand.ctypes.data, score.ctypes.data, L, n_cand, mc, cc.ctypes.data, cs.ctypes.data,
                                steps.ctypes.data, contour.ctypes.data, f0.ctypes.data)
        assert same_bits(steps[4], contour), "FixStep1..4 called one by one differ from FixF0Contour"
        return cc, cs, steps, f0

    def dio_contour(self, cand, score, L, frame_period, fs, f0_floor, allowed_range):
        """cand, score: [nb][stride] -> best[L], f0[L]"""
        cand, score = np.ascontiguousarray(cand), np.ascontiguousarray(score)
        nb, stride = cand.shape
        best, f0 = np.zeros(L), np.zeros(L)
        self.lib.RefDioContour(frame_period, nb, fs, cand.ctypes.data, score.ctypes.data, stride, L, f0_floor,
                               allowed_range, best.ctypes.data, f0.ctypes.data)
        return best, f0


@pytest.fixture(scope="session")
def tail():
    return RefTail()


# ------------------------------------------------------------------ Harvest: one utterance's candidate map
@dataclass
class Map:
    L: int
    nc: int                    # candidates per overlap slot group: nc * 7 slots are used
    rng: tuple                 # (f0_floor, f0_ceil): decides max_cand, i.e. the row stride
    cand: np.ndarray           # [L][nc * 7]
    score: np.ndarray
    name: str = ""


def max_cand(rng):
    return hs.matlab_round(len(hs.band_list(*rng)) / 10.0) * 7


def empty(L, nc, rng=R_DEFAULT, name=""):
    return Map(L, nc, rng, np.zeros((L, nc * 7)), np.zeros((L, nc * 7)), name)


def track(f, i, slot):
    """the value track `slot` holds at frame i: level f with a slow ripple far inside FixStep1's 0.8 %, so that equal
    values identify the track and the frame"""
    return f * (1.0 + 2e-4 * np.sin(0.7 * np.asarray(i, dtype=np.float64) + slot))


def put(m, slot, f, a, b, score):
    """frames a .. b (inclusive) of `slot` carry track f with this score (0: a candidate SearchF0Base never picks but
    ExtendF0 follows)"""
    i = np.arange(max(a, 0), min(b, m.L - 1) + 1)
    m.cand[i, slot] = track(f, i, slot)
    m.score[i, slot] = score
    return m


def runs(v):
    """[(first, last)] of the nonzero runs of v"""
    nz = np.concatenate([[0], (np.asarray(v) != 0).astype(int), [0]])
    d = np.diff(nz)
    return list(zip(np.flatnonzero(d == 1), np.flatnonzero(d == -1) - 1))


def zero_runs(v):
    """lengths of the zero runs between nonzero runs"""
    r = runs(v)
    return [r[k + 1][0] - r[k][1] - 1 for k in range(len(r) - 1)]


# ------------------------------------------------------------------ Harvest: running and comparing
def _env(env):
    class _E:
        def __enter__(self):
            self.saved = {k: os.environ.get(k) for k in env}
            os.environ.update(env)

        def __exit__(self, *a):
            for k, v in self.saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    return _E()


def x_len_for(L):
    return max(1, (FS // 1000) * (L - 1))


def write_refined(path, maps, l1_stride, mcand, stage=3, n=None):
    n = len(maps) if n is None else n
    cand = np.zeros((len(maps), l1_stride, mcand))
    score = np.zeros_like(cand)
    for u, m in enumerate(maps):
        cand[u, :m.L, :m.nc * 7] = m.cand
        score[u, :m.L, :m.nc * 7] = m.score
    with open(path, "wb") as f:
        f.write(b"WBHVDUMP")
        f.write(np.array([1, stage, 0, 0, n, 1, 0, l1_stride, mcand, 0], dtype="<i8").tobytes())
        f.write(struct.pack("<d", float(FS)))
        for ints in ([0] * len(maps), [x_len_for(m.L) for m in maps], [m.L for m in maps], [m.nc for m in maps]):
            f.write(np.array(ints, dtype="<i4").tobytes())
        f.write(cand.tobytes())
        f.write(score.tobytes())


def run_harvest(world, maps, frame_period=5.0, extra_env=None):
    """One harvest call on the batch with the maps loaded in front of harvest_remove_kernel.  Returns per utterance
    (cleaned cand, cleaned score, base, steps[4][L], time_axis, f0)."""
    lens = [x_len_for(m.L) for m in maps]
    x = np.zeros((len(maps), max(lens)))
    l1_stride = int(1000.0 * max(lens) / FS) + 1
    mcand = max(max_cand(m.rng) for m in maps)
    for m in maps:
        assert 1 <= m.nc * 7 <= max_cand(m.rng) and m.cand.shape == (m.L, m.nc * 7)
    with tempfile.TemporaryDirectory() as tmp:
        write_refined(os.path.join(tmp, "load.0"), maps, l1_stride, mcand)
        env = {"WB_LOAD_REFINED": os.path.join(tmp, "load"), "WB_DUMP_CLEANED": os.path.join(tmp, "cleaned"),
               "WB_DUMP_CONTOUR": os.path.join(tmp, "contour")}
        env.update(extra_env or {})
        with _env(env):
            t, f0, fl = world.harvest(pc.make(world, x), FS, hs.options([m.rng for m in maps], frame_period),
                                      x_lengths=lens)
            world.synchronize()
        cl = hs.read_dump(os.path.join(tmp, "cleaned.0"))
        co = hs.read_dump(os.path.join(tmp, "contour.0"))
    assert cl.n == len(maps) and cl.l1_stride == l1_stride and cl.max_cand == mcand
    assert list(cl.l1) == [m.L for m in maps] and list(cl.nc) == [m.nc for m in maps]
    t, f0 = pc.to_np(t), pc.to_np(f0)
    out = []
    for u, m in enumerate(maps):
        n7 = m.nc * 7
        out.append((cl.data[0][u, :m.L, :n7], cl.data[1][u, :m.L, :n7], cl.data[2][u, :m.L], co.data[0][u, :, :m.L],
                    t[u, :fl[u]], f0[u, :fl[u]]))
    return out


# SmoothF0Contour's filter (harvest.cpp:1049-1074, :1081-1084): w_t = x_t + a0 w_(t-1) + a1 w_(t-2), y_t = b0 w_t +
# b1 w_(t-1) + b0 w_(t-2), forward and backward.  The poles are a complex pair of modulus sqrt(0.766) = 0.875, so the
# recursive part's l1 gain is at most 1 / (1 - 0.875)^2 = 64 and |w| <= 64 max|x|.  A step rounds within
# gamma_5 (|x| + (|a0| + |a1|) |w|) <= gamma_5 161 max|x|; carried by that gain and through b (sum|b| = 0.0313) it is
# 0.0313 * 64 * 161 gamma_5 max|x| = 323 gamma_5 max|x| per pass per implementation, and the backward pass (unit DC gain,
# l1 gain of the whole filter below 1.2) carries the forward pass's: 4 * 1.2 * 323 gamma_5 < 9e-13 max|x| in all.
# The library starts each pass 640 samples before the section instead of at the contour's end: a zero-state start
# that far back has decayed by 641 * 0.875^640 < 1e-34 (double pole envelope), nothing beside the rounding term.
SMOOTH_BOUND = 4 * 1.2 * 0.0313 * 64 * 161 * hs.gamma(5) + 1e-34


def subsample(basic, n_frames, frame_period):
    """harvest.cpp:1246-1251"""
    L = len(basic)
    idx = [min(L - 1, hs.matlab_round(i * frame_period / 1000.0 * 1000.0)) for i in range(n_frames)]
    return basic[np.array(idx, dtype=int)] if n_frames else np.zeros(0)


@dataclass
class Report:
    maps: int = 0
    frames: int = 0
    sections: int = 0              # voiced sections FixStep3 extends (its channels)
    merged: int = 0                # ... fewer after MergeF0
    smooth_worst: float = 0.0      # in units of the contour's peak


def compare_harvest(tail, m, got, frame_period, rep=None, what=""):
    """Everything the three kernels leave for one utterance against the reference's functions.  Returns the
    reference's (steps, f0 at 1 ms) for the caller's branch assertions."""
    cc, cs, base, steps, t, f0 = got
    where = f"{what} {m.name} (L {m.L}, nc {m.nc})"
    rc, rs, rsteps, rf0 = tail.harvest_tail(m.cand, m.score, m.nc * 7)
    # RemoveUnreliableCandidates copies or zeroes.  hv_min_rel_error divides once where the reference divides per
    # candidate; division by the positive reference value is monotone under rounding, so the minimum of the rounded
    # quotients is the rounded quotient of the minimum: no candidate may differ, however near 0.05 its error is
    assert same_bits(cc, rc), f"{where}: cleaned candidates differ at {np.argwhere(bits(cc) != bits(rc))[:4].tolist()}"
    assert same_bits(cs, rs), f"{where}: cleaned scores differ at {np.argwhere(bits(cs) != bits(rs))[:4].tolist()}"
    names = ("SearchF0Base", "FixStep1", "FixStep2", "FixStep3", "FixStep4")
    for k, g in enumerate([base] + list(steps)):
        bad = np.flatnonzero(bits(g) != bits(rsteps[k]))
        assert bad.size == 0, (f"{where}: {names[k]} differs at frames {bad[:6].tolist()}: "
                               f"{g[bad[:3]].tolist()} vs {rsteps[k][bad[:3]].tolist()}")
    nf = len(f0)
    want_t = np.array([i * frame_period / 1000.0 for i in range(nf)])
    assert same_bits(t, want_t), f"{where}: time axis"
    want = subsample(rf0, nf, frame_period)
    assert not ((f0 > 0) != (want > 0)).any(), f"{where}: V/UV differs at {np.flatnonzero((f0 > 0) != (want > 0))[:6]}"
    assert np.isfinite(f0).all()
    peak = float(np.max(np.abs(rsteps[4]))) if m.L else 0.0
    err = float(np.max(np.abs(f0 - want))) if nf else 0.0
    assert err <= SMOOTH_BOUND * peak, f"{where}: smoothed f0 off by {err:.3e}, bound {SMOOTH_BOUND * peak:.3e}"
    if rep is not None:
        rep.maps += 1
        rep.frames += m.L
        rep.sections += len(runs(rsteps[2]))
        rep.merged += max(0, len(runs(rsteps[2])) - len(runs(rsteps[3])))
        if peak > 0:
            rep.smooth_worst = max(rep.smooth_worst, err / peak)
    return rsteps, rf0


def check_batch(world, tail, maps, frame_period=5.0, rep=None, what=""):
    got = run_harvest(world, maps, frame_period)
    return [compare_harvest(tail, m, g, frame_period, rep, what) for m, g in zip(maps, got)]


# ------------------------------------------------------------------ Harvest: directed maps
FA, FB, FC = 100.0, 150.0, 225.0     # more than 18 % apart: ExtendF0 never hops from one track to another


def merge_two(a_tail, b_head, dup=0.0, L=400, nc=2):
    """Section A (track FA, slot 0, frames 50 .. 99 at score 5) runs on at score a_tail through frame 140; section B
    (track FB, slot 1, frames 130 .. 199 at score 5) starts at score b_head at frame 90: their extensions overlap in
    90 .. 140 and MergeF0Sub (harvest.cpp:912-932) sums A's scores 10 * 5 + 11 * a_tail against B's 10 * b_head + 11 * 5
    (scores 0 between 100 and 129).  dup: A's values of frames 130 .. 140 once more in slot 5 with this score --
    SearchScore takes the larger."""
    m = empty(L, nc, name=f"merge_two({a_tail},{b_head},{dup})")
    put(m, 0, FA, 50, 99, 5.0); put(m, 0, FA, 100, 129, 0.0); put(m, 0, FA, 130, 140, a_tail)
    put(m, 1, FB, 90, 99, b_head); put(m, 1, FB, 100, 129, 0.0); put(m, 1, FB, 130, 199, 5.0)
    if dup:
        i = np.arange(130, 141)
        m.cand[i, 5] = m.cand[i, 0]
        m.score[i, 5] = dup
    return m


def merge_three(a_tail, b_head, b_tail, c_head):
    """merge_two with a third section C (track FC, slot 2, frames 230 .. 299) overlapping B's extension in 190 .. 240"""
    m = merge_two(a_tail, b_head)
    m.name = f"merge_three({a_tail},{b_head},{b_tail},{c_head})"
    put(m, 1, FB, 200, 229, 0.0); put(m, 1, FB, 230, 240, b_tail)
    put(m, 2, FC, 190, 199, c_head); put(m, 2, FC, 200, 229, 0.0); put(m, 2, FC, 230, 299, 5.0)
    return m


def contained():
    """B's extension (336 .. 364) lies inside A's (51 .. 400): MergeF0Sub returns at once and A's track stays"""
    m = empty(500, 2, name="contained")
    put(m, 0, FA, 50, 299, 5.0); put(m, 0, FA, 300, 400, 0.0)
    put(m, 1, FB, 340, 360, 5.0)
    m.score[340:361, 0] = 1.0
    return m


def sort_quirk():
    """Three sections whose extended starts decrease (A 231, B 220, C 212): MakeSortedOrder as written
    (harvest.cpp:883-896) orders them B, C, A where a sort would give C, B, A, and MergeF0 starts from channel 0 (A)
    and merges order[1] and order[2] only."""
    m = empty(500, 2, name="sort_quirk")
    put(m, 0, FA, 230, 260, 5.0)
    put(m, 1, FB, 220, 269, 0.0); put(m, 1, FB, 270, 300, 5.0)
    put(m, 2, FC, 212, 309, 0.0); put(m, 2, FC, 310, 350, 5.0)
    return m


def dropped_and_running_mean():
    """ExtendSub (harvest.cpp:840-856): a 60 Hz section of 32 frames is dropped (2200 / 60 > 31) and moves the later
    ones down one place; a 100 Hz section with ed - st = 21 is kept only because mean_f0 still holds the 400 Hz of the
    section before it (2200 / ((400 + 21 * 100) / 21) = 18.5 < 21, where 2200 / 100 is not), and one with ed - st = 20
    after a 100 Hz section is dropped (2200 / ((100 + 20 * 100) / 20) = 20.95)."""
    m = empty(700, 1, name="dropped_and_running_mean")
    put(m, 0, 60.0, 20, 51, 5.0)
    put(m, 1, 400.0, 100, 160, 5.0)
    put(m, 2, 100.0, 200, 221, 5.0)       # FixStep1 takes the first frame, ExtendF0 brings it back: st 200, ed 221
    put(m, 3, 100.0, 300, 400, 5.0)
    put(m, 4, 100.0, 500, 520, 5.0)
    return m


def extension_edges(L=160):
    """A's track runs at score 0 from frame 0 to L - 1: ExtendF0 is clipped at frames 1 and L - 2 and writes 0 and L - 1"""
    m = empty(L, 1, name=f"extension_edges({L})")
    put(m, 0, FA, 0, L - 1, 0.0)
    put(m, 0, FA, 60, 99, 5.0)
    return m


def misses():
    """holes of three frames are crossed, the fourth consecutive miss stops ExtendF0 (harvest.cpp:808-815)"""
    m = empty(400, 1, name="misses")
    put(m, 0, FA, 150, 199, 5.0)
    for a, b in ((203, 210), (214, 220), (225, 260), (139, 146), (130, 135), (100, 125)):
        put(m, 0, FA, a, b, 0.0)
    return m


def select_tie():
    """SelectBestF0 (harvest.cpp:636-650) keeps the LAST of the candidates with the smallest error: after a section
    at exactly 100 Hz, 96 Hz (slot 0) and 104 Hz (slot 1) are both 0.04 away and the extension goes on with 104."""
    m = empty(300, 1, name="select_tie")
    m.cand[50:100, 0], m.score[50:100, 0] = 100.0, 5.0
    m.cand[100:120, 0], m.cand[100:120, 1] = 96.0, 104.0
    return m


def short_sections_and_gaps():
    """400 Hz runs of 6 .. 10 base frames (FixStep1 takes the first, FixStep2 keeps ed - st >= 6, i.e. runs of 8 up)
    and, further on, 40-frame runs 6 .. 12 empty frames apart (FixStep4 bridges fewer than 9)"""
    m = empty(1200, 1, name="short_sections_and_gaps")
    pos = 10
    for n in (6, 7, 8, 9, 10, 7, 8):
        put(m, 0, 400.0, pos, pos + n - 1, 5.0)
        pos += n + 30
    for gap in (6, 7, 8, 9, 10, 11, 12, 9, 8):
        put(m, 0, 400.0, pos, pos + 39, 5.0)
        pos += 40 + gap
    assert pos < m.L
    return m


def ties(nc=20):
    """Equal best scores in several slots of a frame: SearchF0Base keeps the first (harvest.cpp:699-703).  140 slots:
    a lane of the warp arg-max holds slots lane, lane + 32, ...; the pairs are in one lane (3, 67), in different lanes
    with the lower slot in the higher lane (37, 67 and 30, 33) and more than 32 apart (8, 104)."""
    m = empty(600, nc, R_WIDE, name="ties")
    for k, (lo, hi) in enumerate(((3, 67), (37, 67), (30, 33), (8, 104), (100, 139))):
        a = 20 + 110 * k
        put(m, lo, 120.0, a, a + 79, 4.0)
        put(m, hi, 200.0, a, a + 79, 4.0)
        put(m, (lo + hi) // 2, 320.0, a, a + 79, 3.0)
    return m


def many_sections(n_sections, L=None):
    """n_sections runs of 12 frames at 400 Hz, 12 empty frames apart: more sections than harvest_smooth_kernel has
    scratch slots (32) or threads (128)"""
    L = L or 24 * n_sections + 30
    m = empty(L, 1, name=f"many_sections({n_sections})")
    for s in range(n_sections):
        put(m, 0, 400.0, 10 + 24 * s, 21 + 24 * s, 5.0)
    return m


def dense_sections(L):
    """The contour that needs the most multi-channel storage: levels of 8 frames alternating between 400 and 440 Hz.
    FixStep1 zeroes the first frame of every level, so FixStep2 sees sections of 7 frames (ed - st = 6, the shortest
    it keeps) one frame apart, and every one extends by the full 101 frames to either side (the levels are 10 %
    apart): each takes 7 + 208 doubles, 26.9 per frame of the utterance."""
    m = empty(L, 1, name=f"dense_sections({L})")
    i = np.arange(L)
    m.cand[:, 0] = np.where((i // 8) % 2 == 0, 400.0, 440.0)
    m.score[:, 0] = 5.0
    return m


def random_map(rng, L=None, wide=None):
    """Piecewise tracks with jitter, drift, octave jumps, dropouts and score-0 stretches in random slots; scores from
    a small set so that ties are common; now and then a value twice in one row with different scores."""
    wide = rng.random() < 0.3 if wide is None else wide
    r = R_WIDE if wide else R_DEFAULT
    nc = int(rng.integers(1, max_cand(r) // 7 + 1))
    L = int(L or rng.integers(3, 3000))
    m = empty(L, nc, r, name="random")
    n7 = nc * 7
    for _ in range(int(rng.integers(1, 6))):
        slot = int(rng.integers(0, n7))
        f = float(rng.uniform(60, 600))
        i = 0
        while i < L:
            seg = int(rng.integers(3, 200))
            kind = rng.random()
            j = min(L, i + seg)
            if kind < 0.25:
                pass                                            # dropout
            else:
                if kind < 0.35:
                    f = f * 2 if f < 300 else f / 2             # octave jump
                elif kind < 0.5:
                    f = float(np.clip(f * rng.uniform(0.8, 1.25), 50, 900))
                k = np.arange(i, j)
                v = f * (1 + rng.uniform(-0.0012, 0.0012, size=j - i)) * (1 + 0.0005 * (k - i) * rng.uniform(-1, 1))
                m.cand[k, slot] = v
                m.score[k, slot] = float(rng.integers(0, 5)) if rng.random() < 0.8 else rng.integers(1, 4, size=j - i)
                if rng.random() < 0.15:
                    s2 = int(rng.integers(0, n7))
                    m.cand[k, s2] = v
                    m.score[k, s2] = float(rng.integers(0, 7))
            if rng.random() < 0.3:
                slot = int(rng.integers(0, n7))
            i = j + (int(rng.integers(0, 14)) if rng.random() < 0.5 else 0)
    return m


# ------------------------------------------------------------------ Harvest: the checks
def check_merge(world, tail):
    """Every outcome of MergeF0Sub on two and on three overlapping sections, the exact tie, SearchScore's maximum over
    equal candidates, a contained section, a section that starts after the merged one, and MakeSortedOrder's order."""
    rep = Report()
    two = [merge_two(2.0, 1.0), merge_two(1.0, 1.0), merge_two(2.5, 2.25), merge_two(1.0, 1.0, dup=3.0)]
    three = [merge_three(a, b, c, d) for a, b in ((2.0, 1.0), (1.0, 1.0)) for c, d in ((2.0, 1.0), (1.0, 1.0))]
    far = empty(900, 1, name="far_apart")
    put(far, 0, FA, 50, 120, 5.0); put(far, 0, FB, 500, 560, 5.0)
    maps = two + three + [contained(), sort_quirk(), far]
    res = check_batch(world, tail, maps, rep=rep, what="merge")
    on = lambda steps, f, slot, i: steps[3][i] == track(f, i, slot)   # FixStep3's frame i carries that track's value
    s = [r[0] for r in res]
    # score1 72 > score2 65: A up to ed1 = 140, B from there
    assert on(s[0], FA, 0, 120) and on(s[0], FA, 0, 139) and on(s[0], FB, 1, 141)
    # 61 < 65: B from st2 = 90
    assert on(s[1], FB, 1, 90) and on(s[1], FB, 1, 120) and on(s[1], FA, 0, 89)
    # 77.5 == 77.5: not greater, B from st2
    assert on(s[2], FB, 1, 90) and on(s[2], FB, 1, 120)
    # as s[1], but the second copy of A's values scores 3: 50 + 33 > 65
    assert on(s[3], FA, 0, 120) and on(s[3], FB, 1, 141)
    for k, (ab, cd) in enumerate([(x, y) for x in (True, False) for y in (True, False)]):
        st = s[4 + k]
        assert on(st, FA if ab else FB, 0 if ab else 1, 120)
        assert on(st, FB if cd else FC, 1 if cd else 2, 220) and on(st, FC, 2, 245)
    assert on(s[8], FA, 0, 350) and s[8][0][350] == track(FB, 350, 1)   # base picked B, the merged contour keeps A
    # the reference's order: C is merged into A (C wins 212 .. 350: A's 5 * 30 against nothing, then ...), B never;
    # a sorted order would merge B first.  What matters here: B's own frames 270 .. 300 end up carrying C or nothing
    q = s[9]
    assert not on(q, FB, 1, 285), "MakeSortedOrder: the reference never merges channel B here"
    assert len(runs(s[10][3])) == 2
    return rep


def check_extend(world, tail):
    rep = Report()
    maps = [dropped_and_running_mean(), extension_edges(160), extension_edges(103), misses(), short_sections_and_gaps(), select_tie()]
    res = check_batch(world, tail, maps, rep=rep, what="extend")
    d = res[0][0][3]
    r = runs(d)
    assert d[30] == 0 and d[130] != 0, "the 60 Hz section is dropped, the 400 Hz one kept"
    assert d[210] != 0 and d[350] != 0 and d[510] == 0, "running mean_f0: kept after 400 Hz, dropped after 100 Hz"
    assert len(r) == 3
    for k in (1, 2):                       # extension_edges: the whole axis is voiced after FixStep3
        e = res[k][0][3]
        assert (e != 0).all(), "ExtendF0 reaches frames 0 and L - 1"
    ms = res[3][0][3]
    assert ms[214] != 0 and ms[211:214].tolist() == [0.0] * 3 and ms[130] != 0, "three misses are crossed"
    assert not ms[221:].any() and not ms[:130].any(), "four misses stop the extension: 225 .. 260, 100 .. 125 unreached"
    sg = res[4][0]
    lens1 = [b - a for a, b in runs(sg[1][:270])]
    assert 5 in lens1 and 6 in lens1, "FixStep1 sections with ed - st of 5 and 6"
    assert sorted(set(b - a for a, b in runs(sg[2][:270]))) == [6, 7, 8], "FixStep2 keeps ed - st >= 6 only"
    g3, g4 = zero_runs(sg[3][300:]), zero_runs(sg[4][300:])
    assert 8 in g3 and 9 in g3 and 8 not in g4 and 9 in g4 and min(g4) == 9, f"FixStep4 bridges gaps below 9: {g3} {g4}"
    tie = res[5][0][3]
    assert tie[99] == 100.0 and (tie[100:120] == 104.0).all(), "SelectBestF0: the last of two equally near candidates"
    return rep


def check_ties_and_counts(world, tail):
    rep = Report()
    maps = [ties(), many_sections(40), many_sections(140), empty(1, 1), empty(2, 1), empty(3, 1),
            put(empty(3, 2), 1, FA, 0, 2, 5.0), put(empty(12, 1), 0, 400.0, 0, 11, 5.0)]
    for m, nm in zip(maps[3:], ("L1", "L2", "L3", "L3_voiced", "L12_voiced")):
        m.name = nm
    res = check_batch(world, tail, maps, rep=rep, what="ties")
    base = res[0][0][0]
    for k, lo in enumerate((3, 37, 30, 8, 100)):
        i = 20 + 110 * k + 40
        assert base[i] == track(120.0, i, lo), "SearchF0Base: the first of two equal scores"
    assert len(runs(res[1][0][4])) == 40 and len(runs(res[2][0][4])) == 140
    return rep


def check_frame_periods(world, tail):
    """the subsampling index min(L - 1, round(t * 1000)) at frame periods that are and are not whole milliseconds"""
    rep = Report()
    rng = np.random.default_rng(5)
    for fp in (1.0, 2.5, 5.0, 5.8):
        maps = [random_map(rng, L=L) for L in (997, 1500, 64)] + [many_sections(40, L=1003)]
        check_batch(world, tail, maps, frame_period=fp, rep=rep, what=f"frame_period {fp}")
    return rep


def check_ragged_batch(world, tail):
    """utterances that differ in L, nc and range group: both strides are larger than most rows"""
    rep = Report()
    rng = np.random.default_rng(6)
    maps = [random_map(rng, L=700, wide=False), ties(), random_map(rng, L=2500, wide=True), merge_two(2.0, 1.0),
            random_map(rng, L=5, wide=False), sort_quirk(), random_map(rng, L=1200, wide=True)]
    check_batch(world, tail, maps, rep=rep, what="ragged")
    return rep


def check_dense(world, tail, L=10000):
    """The densest contour there is, at the length of a 10 s utterance: the multi-channel storage must hold it."""
    rep = Report()
    m = dense_sections(L)
    (steps, _), = check_batch(world, tail, [m], rep=rep, what="dense")
    r2 = runs(steps[2])
    assert len(r2) >= (L - 16) // 8 and set(b - a for a, b in r2[1:-1]) == {6}, "sections of 7 frames, one frame apart"
    assert zero_runs(steps[2])[1:-1] == [1] * (len(r2) - 3)
    return rep


def check_random(world, tail, n_maps, seed, per_call=25):
    rep = Report()
    rng = np.random.default_rng(seed)
    for c in range(0, n_maps, per_call):
        maps = [random_map(rng) for _ in range(min(per_call, n_maps - c))]
        check_batch(world, tail, maps, rep=rep, what=f"random seed {seed} call {c // per_call}")
    return rep


def check_load_errors(world, tail):
    """a load file that does not fit the call is an error that says so, never a silent fallback"""
    m = merge_two(2.0, 1.0)
    lens = [x_len_for(m.L)]
    x = np.zeros((1, lens[0]))
    good = dict(l1_stride=m.L, mcand=max_cand(m.rng))
    cases = [("missing", None, "cannot read"), ("stage", dict(good, stage=2), "stage 3"),
             ("stride", dict(good, l1_stride=m.L + 1), "differ"), ("cand", dict(good, mcand=98), "differ"),
             ("n", dict(good, n=2), "differ")]
    for name, kw, text in cases:
        with tempfile.TemporaryDirectory() as tmp:
            if kw:
                write_refined(os.path.join(tmp, "load.0"), [m], **kw)
            with _env({"WB_LOAD_REFINED": os.path.join(tmp, "load")}):
                with pytest.raises(WorldError, match=text):
                    world.harvest(pc.make(world, x), FS, hs.options([m.rng]), x_lengths=lens)
    with tempfile.TemporaryDirectory() as tmp:       # truncated payload, wrong frame count
        write_refined(os.path.join(tmp, "load.0"), [m], **good)
        with open(os.path.join(tmp, "load.0"), "r+b") as f:
            f.truncate(os.path.getsize(f.name) - 8)
        with _env({"WB_LOAD_REFINED": os.path.join(tmp, "load")}):
            with pytest.raises(WorldError, match="payload"):
                world.harvest(pc.make(world, x), FS, hs.options([m.rng]), x_lengths=lens)
        m2 = empty(m.L - 1, m.nc)
        write_refined(os.path.join(tmp, "load.0"), [m2], **good)
        with _env({"WB_LOAD_REFINED": os.path.join(tmp, "load")}):
            with pytest.raises(WorldError, match="frame counts"):
                world.harvest(pc.make(world, x), FS, hs.options([m.rng]), x_lengths=lens)


def check_wrapper_pin(world, ref, tail, golden):
    """The glue of RefHarvestTail (row layout, number_of_candidates = nc * 7): fed the library's own refined candidates
    of the golden utterance it must reproduce the reference's Harvest.  The refined candidates carry the REFINED
    stage's rounding (harvest_stages_common.refine_one: below 1e-9 relative), the decision stages select among them
    and the smoothing filter has unit gain, so voiced frames agree within 1e-6 wherever both decide the same; the
    reference's own decisions may differ only where a candidate sits within that of a threshold."""
    x, fs = pc.wav_from_golden(golden)
    d = hs.capture(world, x[None, :], fs, [R_DEFAULT], [len(x)])["REFINED"][0]
    L, nc = int(d.l1[0]), int(d.nc[0])
    _, _, _, f0_1ms = tail.harvest_tail(d.data[0][0, :L], d.data[1][0, :L], nc * 7)
    t, want = ref.harvest(x, fs)
    got = subsample(f0_1ms, len(want), 5.0)
    assert (want > 0).sum() > 50
    flips = int(((got > 0) != (want > 0)).sum())
    assert flips == 0, f"{flips} V/UV differences"
    v = want > 0
    assert np.max(np.abs(got[v] - want[v]) / want[v]) < 1e-6


# ------------------------------------------------------------------ DIO
def dio_bands(opt):
    """number_of_bands (dio.cpp:582-583)"""
    return 1 + int(math.log(opt.f0_ceil / opt.f0_floor) / math.log(2.0) * opt.channels_in_octave)


def dio_vrm(frame_period, f0_floor):
    return int(0.5 + 1000.0 / frame_period / f0_floor) * 2 + 1


def dio_option(world, f0_floor=71.0, f0_ceil=800.0, frame_period=5.0, allowed_range=0.1, channels=2.0):
    o = world.dio_option()
    o.f0_floor, o.f0_ceil, o.frame_period, o.allowed_range, o.channels_in_octave = (f0_floor, f0_ceil, frame_period,
                                                                                   allowed_range, channels)
    return o


def dio_random(rng, L, nb):
    """per band a piecewise track with jitter and zeros; scores and now and then candidates from small sets, so that
    the best-score scan and SelectBestF0's nearest candidate meet exact ties"""
    cand, score = np.zeros((nb, L)), np.zeros((nb, L))
    f = float(rng.uniform(80, 400))
    for b in range(nb):
        i = 0
        while i < L:
            j = min(L, i + int(rng.integers(2, 80)))
            kind = rng.random()
            if kind < 0.2:
                f = float(rng.uniform(80, 400))
            base = f * (2.0 if kind > 0.9 else 1.0)
            if kind < 0.1:
                cand[b, i:j] = 0.0
            elif kind < 0.3:
                cand[b, i:j] = float(round(base))                      # exact repeats across bands
            else:
                cand[b, i:j] = base * (1 + rng.uniform(-0.02, 0.02, size=j - i))
            score[b, i:j] = rng.integers(0, 4, size=j - i) * 0.25 if rng.random() < 0.7 else rng.uniform(0, 1)
            i = j
    # symmetric ties of SelectBestF0: two bands at reference -+ d
    return cand, score


def run_dio(world, cases, frame_period):
    """cases: [(option, L, cand[nb][L], score)].  One dio call with the rows loaded in front of dio_contour_kernel."""
    per_ms = FS / 1000.0
    lens = [max(1, int(math.ceil((L - 1) * frame_period * per_ms))) for _, L, _, _ in cases]
    for (o, L, _, _), n in zip(cases, lens):
        assert world.frames(FS, n, frame_period) == L, (L, n)
    x = np.zeros((len(cases), max(lens)))
    fstr = max(L for _, L, _, _ in cases)
    nb = max(dio_bands(o) for o, _, _, _ in cases)
    cand, score = np.zeros((len(cases), nb, fstr)), np.zeros((len(cases), nb, fstr))
    for u, (o, L, c, s) in enumerate(cases):
        assert c.shape == (dio_bands(o), L)
        cand[u, :c.shape[0], :L], score[u, :c.shape[0], :L] = c, s
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "cand.0"), "wb") as f:
            f.write(b"WBDICAND")
            f.write(np.array([1, 0, len(cases), nb, fstr], dtype="<i8").tobytes())
            f.write(cand.tobytes())
            f.write(score.tobytes())
        with _env({"WB_LOAD_DIO_CAND": os.path.join(tmp, "cand")}):
            opts = [o for o, _, _, _ in cases]
            t, f0, fl = world.dio(pc.make(world, x), FS, opts if len(opts) > 1 else opts[0], x_lengths=lens)
            world.synchronize()
    return pc.to_np(t), pc.to_np(f0), fl


def check_dio(world, tail, seed=11):
    """dio_contour_kernel on loaded rows: L below, at and above the minimum voiced range, several range groups and
    allowed ranges in one batch (the group's band count below the row count, L below the frame stride), frame periods
    that change the minimum range.  Selections only: bit for bit."""
    rng = np.random.default_rng(seed)
    compared = voiced = 0
    for fp in (5.0, 1.0, 2.5, 5.8):
        o1 = dio_option(world, 71.0, 800.0, fp, 0.1)
        o2 = dio_option(world, 40.0, 1100.0, fp, 0.25, channels=3.0)
        o3 = dio_option(world, 120.0, 600.0, fp, 0.02)
        cases = []
        for o in (o1, o2, o3):
            vrm = dio_vrm(fp, o.f0_floor)
            for L in (vrm - 1, vrm, vrm + 1, 2 * vrm + 3, int(rng.integers(200, 1500))):
                if L >= 1:
                    cases.append((o, L) + dio_random(rng, L, dio_bands(o)))
        t, f0, fl = run_dio(world, cases, fp)
        for u, (o, L, c, s) in enumerate(cases):
            assert fl[u] == L
            best, want = tail.dio_contour(c, s, L, fp, FS, o.f0_floor, o.allowed_range)
            where = f"dio fp {fp} utterance {u} (L {L}, vrm {dio_vrm(fp, o.f0_floor)}, {c.shape[0]} bands)"
            bad = np.flatnonzero(bits(f0[u, :L]) != bits(want))
            assert bad.size == 0, f"{where}: f0 differs at {bad[:6].tolist()}"
            assert same_bits(t[u, :L], np.array([i * fp / 1000.0 for i in range(L)])), where
            compared += L
            voiced += int((want > 0).sum())
    assert voiced > 500, "the maps must leave voiced sections to extend"
    # a single option through the batch-wide call, and the load file's checks
    o = dio_option(world)
    c, s = dio_random(rng, 300, dio_bands(o))
    t, f0, fl = run_dio(world, [(o, 300, c, s)], 5.0)
    assert same_bits(f0[0, :300], tail.dio_contour(c, s, 300, 5.0, FS, o.f0_floor, o.allowed_range)[1])
    with tempfile.TemporaryDirectory() as tmp:
        with _env({"WB_LOAD_DIO_CAND": os.path.join(tmp, "none")}):
            with pytest.raises(WorldError, match="cannot read"):
                world.dio(pc.make(world, np.zeros((1, 2000))), FS, o)
        with open(os.path.join(tmp, "bad.0"), "wb") as f:
            f.write(b"WBDICAND" + np.array([1, 0, 1, 3, 7], dtype="<i8").tobytes())
        with _env({"WB_LOAD_DIO_CAND": os.path.join(tmp, "bad")}):
            with pytest.raises(WorldError, match="differ"):
                world.dio(pc.make(world, np.zeros((1, 2000))), FS, o)
    return compared, voiced
