"""Harvest checked stage by stage: each stage of the library is fed the library's own previous-stage output (captured
through the WB_DUMP_* test hooks of wb_harvest.cu) and compared with an extended-precision numpy restatement of the
reference's code for that stage, written from harvest.cpp (line numbers below).  Every tolerance is a propagated
rounding bound; decisions that sit within their bound of a threshold are excluded and counted, never guessed.
The same checks run on the host emulation (CPU) and on the CUDA library (-m gpu)."""
import ctypes as C
import glob
import math
import os
import tempfile
from dataclasses import dataclass, field

import numpy as np
import pytest

import test_parity_common as pc
from world_b200.api import HarvestOption

LD = np.longdouble
U = 2.0 ** -53                       # unit roundoff of float64
PI = LD("3.14159265358979323846264338327950288")
STAGES = ("DECIMATED", "RAW", "BASE", "REFINED")
WB_HV_BASE = 32


def gamma(n):
    """gamma_n = n u / (1 - n u): the bound on the relative error of any n-term float64 sum or product chain."""
    return n * U / (1.0 - n * U)


def require_extended():
    if np.finfo(LD).nmant < 63:
        pytest.skip(f"np.longdouble has {np.finfo(LD).nmant} mantissa bits here; the restatements need 63")


def matlab_round(v):
    return int(v + 0.5) if v > 0 else int(v - 0.5)


# ------------------------------------------------------------------ capture
@dataclass
class Dump:
    stage: int
    chunk: int
    u0: int
    n: int
    ratio: int
    nb: int
    l1_stride: int
    max_cand: int
    afs: float
    ugrp: np.ndarray
    y_len: np.ndarray
    l1: np.ndarray
    nc: np.ndarray
    groups: list                          # [(nb, f0_floor, f0_ceil)]
    data: list = field(default_factory=list)


def read_dump(path):
    b = open(path, "rb").read()
    assert b[:8] == b"WBHVDUMP", path
    ver, stage, chunk, u0, n, ratio, nb, l1s, maxc, ng = (int(v) for v in np.frombuffer(b, "<i8", 10, 8))
    assert ver == 1
    o = 88
    afs = float(np.frombuffer(b, "<f8", 1, o)[0]); o += 8
    ints = []
    for _ in range(4):
        ints.append(np.frombuffer(b, "<i4", n, o).copy()); o += 4 * n
    groups = []
    for _ in range(ng):
        gnb = int(np.frombuffer(b, "<i4", 1, o)[0])
        lo, hi = np.frombuffer(b, "<f8", 2, o + 4)
        groups.append((gnb, float(lo), float(hi))); o += 20
    d = Dump(stage, chunk, u0, n, ratio, nb, l1s, maxc, afs, *ints, groups)
    if stage == 0:
        for u in range(n):
            d.data.append(np.frombuffer(b, "<f8", int(d.y_len[u]), o).copy()); o += 8 * int(d.y_len[u])
    elif stage == 1:
        d.data.append(np.frombuffer(b, "<f8", n * nb * l1s, o).reshape(n, nb, l1s).copy()); o += 8 * n * nb * l1s
    elif stage == 2:
        d.data.append(np.frombuffer(b, "<f8", n * l1s * WB_HV_BASE, o).reshape(n, l1s, WB_HV_BASE).copy())
        o += 8 * n * l1s * WB_HV_BASE
        d.data.append(np.frombuffer(b, "<i4", n * l1s, o).reshape(n, l1s).copy()); o += 4 * n * l1s
    else:
        for _ in range(2):
            d.data.append(np.frombuffer(b, "<f8", n * l1s * maxc, o).reshape(n, l1s, maxc).copy())
            o += 8 * n * l1s * maxc
    assert o == len(b), f"{path}: {len(b) - o} trailing bytes"
    return d


def options(ranges, frame_period=5.0):
    out = []
    for lo, hi in ranges:
        o = HarvestOption()
        o.f0_floor, o.f0_ceil, o.frame_period = lo, hi, frame_period
        out.append(o)
    return out


def capture(world, x, fs, ranges, lens, env=None):
    """Runs the batch once with every stage hook set (plus `env`); returns {stage name: [Dump per chunk]}."""
    env = dict(env or {})
    with tempfile.TemporaryDirectory() as tmp:
        for s in STAGES:
            env["WB_DUMP_" + s] = os.path.join(tmp, s.lower())
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            world.harvest(pc.make(world, x), fs, options(ranges), x_lengths=lens)
            world.synchronize()
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        out = {}
        for s in STAGES:
            files = glob.glob(os.path.join(tmp, s.lower()) + ".*")
            out[s] = sorted((read_dump(f) for f in files), key=lambda d: d.chunk)
    return out


# ------------------------------------------------------------------ a. decimation (harvest.cpp:43-93)
def decimated_reference(ref, x, ratio):
    """GetWaveformAndSpectrumSub + DC removal (harvest.cpp:43-66, :81-85) with the reference's own decimate; the
    mean is exact (fsum) so the comparison carries only the device's own rounding of it."""
    n = len(x)
    ylen = int(math.ceil(n / ratio))
    if ratio == 1:
        dec = np.array(x, dtype=np.float64)
    else:
        lag = int(math.ceil(140.0 / ratio) * ratio)
        xp = np.concatenate([np.full(lag, x[0]), x, np.full(lag, x[-1])])
        out = np.zeros(len(xp))   # decimate writes up to 9 / ratio samples past (n - 1) / ratio + 1; harvest.cpp:53
        ref.lib.decimate.restype = None
        ref.lib.decimate.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        ref.lib.decimate(xp.ctypes.data, len(xp), ratio, out.ctypes.data)
        dec = out[lag // ratio: lag // ratio + ylen]
    mean = LD(math.fsum(dec)) / ylen
    return dec, (dec.astype(LD) - mean)


def check_decimated(dumps, ref, x, lens):
    """Bound per sample.  One pass of the decimation IIR w_i = x_i + sum a_k w_(i-k), y_i = sum b_k w_(i-k)
    (matlabfunctions.cpp:115-124) rounds each recursion step within gamma_6 (|x| + sum|a| |w|), which its recursive
    part carries with l1 gain G_a, while |w| <= G_a |x|; the output adds sum|b| times that plus gamma_7 sum|b| |w|.
    The backward pass carries the forward pass's error with the l1 gain G of the whole filter (< 1.51) and adds
    its own.  Over the reference's coefficient tables (ratios 2 .. 12; worst at 12: G_a = 77.6, sum|a| = 5.26,
    sum|b| = 0.0169) this is < 1250 gamma_6 of the input peak per implementation.  The reference's sequential
    passes and the device's 256-sample blocks after a 512-sample run-in (DESIGN 3 item 6; state error below
    0.889^512 = 7e-27 of the peak) err independently: 2500 gamma_6 = 1.7e-12 of the peak.  The device's mean is a
    sum in some order of ylen values, within gamma_ylen mean|y| of the exact one used here, and the subtraction
    rounds by u.  Returns the worst error in units of the row peak."""
    worst = 0.0
    for d in dumps:
        for i in range(d.n):
            u = d.u0 + i
            xu = x[u, :lens[u]]
            dec, want = decimated_reference(ref, xu, d.ratio)
            got = d.data[i]
            assert len(got) == len(want)
            peak = float(np.max(np.abs(dec)))
            e_dec = 0.0 if d.ratio == 1 else 2500 * gamma(6) * float(np.max(np.abs(xu)))
            bound = e_dec + gamma(len(dec)) * float(np.mean(np.abs(dec))) + 2 * U * np.abs(got)
            err = np.abs(got.astype(LD) - want).astype(np.float64)
            assert (err <= bound).all(), \
                f"decimated row {u}: error {err.max():.3e} > bound at sample {int(np.argmax(err - bound))}"
            worst = max(worst, float(err.max()) / peak)
    return worst


# ------------------------------------------------------------------ b. raw candidate map (harvest.cpp:99-343)
def band_list(f0_floor, f0_ceil):
    """boundary_f0_list (harvest.cpp:1149-1157), channels_in_octave 40"""
    lo, hi = f0_floor * 0.9, f0_ceil * 1.1
    nb = 1 + int(math.log(hi / lo) / math.log(2.0) * 40)
    return [lo * 2.0 ** ((i + 1) / 40.0) for i in range(nb)]


def band_taps(boundary, afs):
    """GetFilteredSignal's filter (harvest.cpp:101-106) in float64 exactly as the reference rounds it (NuttallWindow,
    common.cpp), element by element through the C library's cos."""
    lh = matlab_round(afs / boundary * 2.0)
    n = 2 * lh + 1
    h = np.empty(n)
    for i in range(n):
        t = i / (n - 1.0)
        w = (0.355768 - 0.487396 * math.cos(2.0 * math.pi * t) + 0.144232 * math.cos(4.0 * math.pi * t)
             - 0.012604 * math.cos(6.0 * math.pi * t))
        h[i] = w * math.cos(2 * math.pi * boundary * (i - lh) / afs)
    return h, lh


def _ripple(y, h, lh, fft_size):
    """The reference's mirroring loop (harvest.cpp:122-133) also stores product bin i in slot N - i - 1; for
    i = N/2 - 1 and N/2 those slots are inside the half its c2r reads, so both bins end up as Q = Y[N/2] Z1, with
    Z1 = Y[N/2-1] H[N/2-1], instead of Z1 and Y[N/2] H[N/2].  Normalised to the linear convolution, output sample m
    gains (2 Re((Q - Z1) e^(j 2 pi (N/2-1) m / N)) + (Re Q - Y[N/2] H[N/2]) (-1)^m) / N; index_bias = lh + 1
    (:140-142)."""
    N = fft_size
    n = np.arange(N, dtype=LD)
    yl = np.zeros(N, dtype=LD); yl[:len(y)] = y
    hl = np.zeros(N, dtype=LD); hl[:len(h)] = h
    ang = -2 * PI * (N // 2 - 1) * n / N
    c, s = np.cos(ang), np.sin(ang)
    yr, yi = np.sum(yl * c), np.sum(yl * s)
    hr, hi = np.sum(hl * c), np.sum(hl * s)
    zr, zi = yr * hr - yi * hi, yr * hi + yi * hr
    sgn = np.where(n % 2 == 0, LD(1), LD(-1))
    yn, hn = np.sum(yl * sgn), np.sum(hl * sgn)
    qr, qi = yn * zr, yn * zi
    m = (np.arange(len(y)) + lh + 1).astype(LD)
    a = 2 * PI * (N // 2 - 1) * m / N
    return (2 * ((qr - zr) * np.cos(a) - (qi - zi) * np.sin(a)) + (qr - yn * hn) * np.where(m % 2 == 0, 1, -1)) / N


@dataclass
class Train:
    fine: np.ndarray      # fine edges (samples), long double
    dfine: np.ndarray     # bound on the device's error in each
    amb: np.ndarray       # sample positions of crossings whose presence is ambiguous


def _train(f, e):
    """ZeroCrossingEngine (harvest.cpp:162-197) on the train f (long double) whose device values are within e."""
    a, b = f[:-1], f[1:]
    ea, eb = e[:-1], e[1:]
    edge = np.nonzero((a > 0) & (b <= 0))[0] + 1
    amb = np.nonzero((a > -ea) & (b <= eb) & ((np.abs(a) <= ea) | (np.abs(b) <= eb)))[0] + 1
    fa, fb = f[edge - 1], f[edge]
    d = fb - fa
    q = fa / d
    fine = edge - q
    ad = np.maximum(np.abs(d).astype(np.float64) - e[edge] - e[edge - 1], 1e-300)
    dq = (e[edge - 1] * np.abs(d).astype(np.float64) + np.abs(fa).astype(np.float64) * (e[edge] + e[edge - 1])) / ad ** 2
    dfine = dq + 4 * U * (np.abs(fine) + np.abs(q)).astype(np.float64)
    return Train(fine, dfine, amb)


def _interp(tr, afs, tq):
    """intervals / locations (:188-191) and interp1 onto the 1 ms grid (matlabfunctions.cpp:136-176); returns the
    values, their bounds and a mask of frames whose interval reads a point next to an ambiguous crossing."""
    fe, de = tr.fine, tr.dfine
    gap = fe[1:] - fe[:-1]
    y = afs / gap
    x = (fe[:-1] + fe[1:]) / 2 / afs
    g = gap.astype(np.float64)
    dy = afs * (de[:-1] + de[1:]) / np.maximum(g - de[:-1] - de[1:], 1e-300) ** 2 + 3 * U * np.abs(y).astype(np.float64)
    dx = (de[:-1] + de[1:]) / 2 / afs + 3 * U * np.abs(x).astype(np.float64)
    m = len(x)
    xd = x.astype(np.float64)
    c = np.clip(np.searchsorted(xd, tq, side="right"), 1, m - 1)
    x0, x1, y0, y1 = x[c - 1], x[c], y[c - 1], y[c]
    s = (tq.astype(LD) - x0) / (x1 - x0)
    val = y0 + s * (y1 - y0)
    sf = np.abs(s).astype(np.float64)
    h = (x1 - x0).astype(np.float64)
    ds = (dx[c - 1] * (1 + sf) + dx[c] * sf) / np.maximum(h - dx[c - 1] - dx[c], 1e-300) + 3 * U * sf
    yd = np.abs(y1 - y0).astype(np.float64)
    bound = np.abs(1 - sf) * dy[c - 1] + sf * dy[c] + yd * ds + 4 * U * (np.abs(y0) + np.abs(s * (y1 - y0))).astype(np.float64)
    # the other side of a knot the query sits on within its bound: linear interpolation is continuous there
    near = (np.abs(tq - xd[c]) <= dx[c]) | (np.abs(tq - xd[c - 1]) <= dx[c - 1])
    ydiff = np.abs(np.diff(y).astype(np.float64))
    nb_diff = np.maximum(ydiff[np.clip(c - 2, 0, m - 2)], ydiff[np.clip(c, 0, m - 2)])
    bound = bound + np.where(near, 2 * (dx[c] + dx[c - 1]) / np.maximum(h, 1e-300) * nb_diff, 0.0)
    excl = np.zeros(len(tq), bool)
    fed = fe.astype(np.float64)
    for p in tr.amb:
        j = int(np.searchsorted(fed, p))
        lo = -np.inf if j - 2 < 0 else fed[j - 2] / afs
        hi = np.inf if j + 2 >= len(fed) else fed[j + 2] / afs
        excl |= (tq >= lo) & (tq <= hi)
    return val, bound, excl


def band_candidates(y, boundary, afs, f0_floor, f0_ceil, l1, fft_size, ripple_in_device):
    """GetF0CandidateFromRawEvent (harvest.cpp:312-329) for one band, in long double.  Returns the candidate row, its
    bound and the excluded frames."""
    h, lh = band_taps(boundary, afs)
    yl = y.astype(LD)
    full = np.convolve(yl, h.astype(LD))
    s = full[lh + 1: lh + 1 + len(y)]                     # delay compensation (:140-142)
    if len(s) < len(y):
        s = np.concatenate([s, np.zeros(len(y) - len(s), LD)])
    rip = _ripple(y, h, lh, fft_size)
    # the device's filtered sample: any order of its K products and sums (gamma_K sum |y||h|); at the decimated
    # rates it omits the reference's ripple, which then belongs to the bound
    mag = np.convolve(np.abs(y), np.abs(h))[lh + 1: lh + 1 + len(y)]
    if len(mag) < len(y):
        mag = np.concatenate([mag, np.zeros(len(y) - len(mag))])
    e = gamma(len(h) + 2) * mag
    if ripple_in_device:
        s = s + rip
        e = e + 8 * U * np.abs(rip).astype(np.float64)
    else:
        e = e + np.abs(rip).astype(np.float64)
    dif = s[1:] - s[:-1]
    ed = e[1:] + e[:-1] + U * np.abs(dif).astype(np.float64)
    trains = [_train(s, e), _train(-s, e), _train(dif, ed), _train(-dif, ed)]
    tq = np.arange(l1) * 1 / 1000.0
    # CheckEvent (:263-269): every train needs more than two intervals; if an ambiguous crossing could move a
    # train across that line, the whole band is excluded
    intervals = [max(len(t.fine) - 1, 0) for t in trains]
    if any(len(t.amb) and v - len(t.amb) <= 2 < v + len(t.amb) for t, v in zip(trains, intervals)):
        return np.zeros(l1), np.zeros(l1), np.ones(l1, bool)
    if min(intervals) <= 2:
        return np.zeros(l1), np.zeros(l1), np.zeros(l1, bool)
    vals, bnds, excl = zip(*(_interp(t, afs, tq) for t in trains))
    cand = (vals[0] + vals[1] + vals[2] + vals[3]) / 4
    cb = sum(bnds) / 4 + 3 * U * sum(np.abs(v) for v in vals).astype(np.float64) / 4
    ex = excl[0] | excl[1] | excl[2] | excl[3]
    cf = cand.astype(np.float64)
    for thr in (boundary * 1.1, boundary * 0.9, f0_ceil, f0_floor):   # GetF0CandidateContourSub (:240-254)
        ex |= np.abs(cf - thr) <= cb
    keep = ~((cf > boundary * 1.1) | (cf < boundary * 0.9) | (cf > f0_ceil) | (cf < f0_floor))
    return np.where(keep, cf, 0.0), np.where(keep, cb, 0.0), ex


@dataclass
class StageReport:
    worst: float = 0.0            # worst error / |value| over the compared entries
    worst_bound: float = 0.0      # largest bound / |value| used
    compared: int = 0
    excluded: int = 0


def check_raw(dec_dumps, raw_dumps):
    """The device's raw candidate map against the restatement from the device's own decimated rows."""
    rep = StageReport()
    assert len(dec_dumps) == len(raw_dumps)
    for dd, rd in zip(dec_dumps, raw_dumps):
        raw = rd.data[0]
        for i in range(rd.n):
            y = dd.data[i]
            gnb, f0_floor, f0_ceil = rd.groups[int(rd.ugrp[i])]
            bl = band_list(f0_floor, f0_ceil)
            assert len(bl) == gnb
            l1 = int(rd.l1[i])
            fft_size = int(2.0 ** (int(math.log(len(y) + 5 + 2 * int(2.0 * rd.afs / bl[0])) / math.log(2.0)) + 1))
            n_ex = 0
            for j, b in enumerate(bl):
                want, bound, ex = band_candidates(y, b, rd.afs, f0_floor, f0_ceil, l1, fft_size, rd.ratio == 1)
                got = raw[i, j, :l1]
                n_ex += int(ex.sum())
                k = ~ex
                bad = k & ((got > 0) != (want > 0))
                assert not bad.any(), \
                    f"utterance {rd.u0 + i} band {j} ({b:.2f} Hz): zero pattern differs at frame {int(np.argmax(bad))}"
                err = np.abs(got - want)
                assert (err[k] <= bound[k]).all(), \
                    f"utterance {rd.u0 + i} band {j}: error {err[k].max():.3e} > bound at frame " \
                    f"{int(np.flatnonzero(k)[np.argmax(err[k] - bound[k])])}"
                nz = k & (want > 0)
                if nz.any():
                    rep.worst = max(rep.worst, float((err[nz] / want[nz]).max()))
                    rep.worst_bound = max(rep.worst_bound, float((bound[nz] / want[nz]).max()))
                rep.compared += int(k.sum())
            assert n_ex <= 0.01 * gnb * l1, f"utterance {rd.u0 + i}: {n_ex} of {gnb * l1} (band, frame) excluded"
            rep.excluded += n_ex
    return rep


# ------------------------------------------------------------------ c. base candidates (harvest.cpp:348-412)
def check_base(raw_dumps, base_dumps):
    """DetectOfficialF0Candidates restated from the device's raw map.  The device sums each section's bands in
    band order like the reference (:374-376), so the base candidates must agree bit for bit; so must the counts
    and nc, the batch-row maximum count."""
    n_cmp = 0
    for rd, bd in zip(raw_dumps, base_dumps):
        base, cnt = bd.data
        for i in range(rd.n):
            gnb = rd.groups[int(rd.ugrp[i])][0]
            l1 = int(rd.l1[i])
            raw = rd.data[0][i, :gnb, :l1]
            vuv = (raw > 0).astype(int)
            vuv[0] = vuv[gnb - 1] = 0
            want = np.zeros((l1, WB_HV_BASE))
            wcnt = np.zeros(l1, int)
            st = np.zeros(l1, int)
            acc = np.zeros(l1)
            for j in range(1, gnb):
                dv = vuv[j] - vuv[j - 1]
                start = dv == 1
                st[start] = j
                acc[start] = 0.0
                close = (dv == -1) & (j - st >= 10)
                for k in np.flatnonzero(close):
                    want[k, wcnt[k]] = acc[k] / (j - st[k])
                    wcnt[k] += 1
                acc = np.where(vuv[j] == 1, acc + raw[j], acc)
            assert np.array_equal(cnt[i, :l1], wcnt), f"utterance {rd.u0 + i}: base candidate counts"
            assert np.array_equal(base[i, :l1], want), \
                f"utterance {rd.u0 + i}: base candidates differ at frame {int(np.argmax((base[i, :l1] != want).any(1)))}"
            assert int(bd.nc[i]) == int(wcnt.max(initial=0)), f"utterance {rd.u0 + i}: nc"
            n_cmp += int(wcnt.sum())
    return n_cmp


# ------------------------------------------------------------------ d. refinement (harvest.cpp:417-631)
def _near_half(v, ulps=8):
    """v within `ulps` of a rounding boundary of matlab_round (k + 1/2) or of int() truncation (an integer)"""
    tol = ulps * U * max(abs(v), 1.0)
    return abs(v - math.floor(v) - 0.5) <= tol or abs(v - round(v)) <= tol


def refine_one(y, afs, k, f, f0_floor, f0_ceil):
    """GetRefinedF0 (:589-617) for candidate f at 1 ms frame k, as a direct long-double DFT at the bins FixF0 reads
    (:507-536).  Returns (refined f0, score, f0 bound, score bound, excluded), where the bounds cover the device's
    double evaluation in any summation order: |dX| <= (gamma_nwin + twiddle chain + window error) sum |x||w|."""
    ylen = len(y)
    hv = 1.5 * afs / f + 1.0
    h = int(hv)
    nwin = 2 * h + 1
    nfft = int(2.0 ** (2.0 + int(math.log(h * 2.0 + 1.0) / math.log(2.0))))
    H = min(int(afs / 2.0 / f), 6)
    binv = [f * nfft / afs * (m + 1) for m in range(H)]
    excluded = _near_half(hv) or any(_near_half(b) for b in binv)
    t = k * 1 / 1000.0
    T = LD(2.0 * h + 1.0) / LD(afs)
    basic = matlab_round((t + (-h + 0) / afs) * afs + 0.001)                      # GetBaseIndex (:434-441)
    idx = basic + np.arange(nwin)
    tmp = (idx.astype(LD) - 1) / LD(afs) - LD(t)                                  # GetMainWindow (:446-456)
    w = LD(0.42) + LD(0.5) * np.cos(2 * PI * tmp / T) + LD(0.08) * np.cos(4 * PI * tmp / T)
    dw = np.empty(nwin, LD)                                                      # GetDiffWindow (:462-468)
    dw[0] = -w[1] / 2
    dw[1:-1] = -(w[2:] - w[:-2]) / 2
    dw[-1] = w[-2] / 2
    xs = y[np.clip(idx - 1, 0, ylen - 1)].astype(LD)                             # GetSpectra (:479-486)
    # the device's window: rounding of its own evaluation, plus the time argument in double ((i - h - 1) / afs in
    # the chain kernel, DESIGN 3 decision 7; ((basic + j) - 1) / afs - t in the per-frame one): both within
    # 2u (t + |basic + j| / afs) of the exact argument, times the window's slope 2 pi / T (0.5 + 0.16)
    slope = float(2 * PI / T) * 0.66
    werr = 16 * U + slope * 2 * U * (t + np.abs(idx).astype(np.float64) / afs)
    steps = nwin // 8 + 2
    xa = np.abs(xs).astype(np.float64)
    num = den = sc = LD(0)
    bnum = bden = bsc = 0.0
    terms = []
    for m in range(H):
        b = matlab_round(binv[m])
        ang = -2 * PI * b * np.arange(nwin, dtype=LD) / nfft
        cs, sn = np.cos(ang), np.sin(ang)
        mr, mi = np.sum(xs * w * cs), np.sum(xs * w * sn)
        dr, di = np.sum(xs * dw * cs), np.sum(xs * dw * sn)
        ex = (gamma(nwin + 2) + 8 * steps * U) * float(np.sum(xa * np.abs(w).astype(np.float64))) + float(np.sum(xa * werr))
        ed = (gamma(nwin + 2) + 8 * steps * U) * float(np.sum(xa * np.abs(dw).astype(np.float64))) + \
            float(np.sum(xa * 2 * werr))
        nm = mr * di - mi * dr
        pw = mr * mr + mi * mi
        X, D = float(np.hypot(float(mr), float(mi))), float(np.hypot(float(dr), float(di)))
        e_nm = 2 * (ex * (D + ed) + X * ed) + 4 * U * float(abs(mr * di) + abs(mi * dr))
        e_pw = 2 * ex * (2 * X + ex) + 4 * U * float(pw)
        pwf = float(pw)
        if pwf == 0.0:
            return 0.0, 0.0, 0.0, 0.0, True
        q = nm / pw
        e_q = (e_nm + float(abs(q)) * e_pw) / max(pwf - e_pw, 1e-300)
        inst = LD(b) * LD(afs) / nfft + q * LD(afs) / 2 / PI
        e_inst = afs / 2 / math.pi * e_q + 6 * U * float(abs(inst) + abs(q * LD(afs)))
        amp = np.sqrt(pw)
        e_amp = e_pw / (2 * math.sqrt(max(pwf - e_pw, 1e-300))) + U * float(amp)
        num += amp * inst
        den += amp * (m + 1)
        sc += abs((inst / (m + 1) - LD(f)) / LD(f))
        bnum += e_amp * float(abs(inst)) + float(amp) * e_inst
        bden += e_amp * (m + 1)
        bsc += e_inst / (m + 1) / f + 4 * U * float(abs(inst / (m + 1) - LD(f)) / LD(f) + 1)
        terms.append(inst)
    rf = num / (den + LD(1e-12))
    rs = 1 / (sc / H + LD(1e-12))
    rff, rsf = float(rf), float(rs)
    denf = float(den)
    e_rf = (bnum + abs(rff) * bden) / max(denf - bden, 1e-300) + 4 * U * abs(rff) + 2 * H * U * (float(abs(num)) / denf)
    e_rs = rsf * rsf * (bsc / H + 2 * H * U * float(sc) / H) / max(1 - rsf * (bsc / H), 1e-300) + 3 * U * rsf
    # the floor / ceiling / score tests (:610-614)
    if abs(rff - f0_floor) <= e_rf or abs(rff - f0_ceil) <= e_rf or abs(rsf - 2.5) <= e_rs:
        excluded = True
    if rff < f0_floor or rff > f0_ceil or rsf < 2.5:
        return 0.0, 0.0, 0.0, 0.0, excluded
    return rff, rsf, e_rf, e_rs, excluded


def overlapped(base_row_frames, nc, k, s, l1):
    """OverlapF0Candidates (:417-429): slot s of frame k"""
    g, j = divmod(s, nc)
    src = k if g == 0 else (k - g if g <= 3 else k + (g - 3))
    if src < 0 or src >= l1:
        return 0.0
    return float(base_row_frames[src, j])


def check_refined(dec_dumps, base_dumps, ref_dumps, frame_step=1):
    """Every (frame, slot) with a nonzero overlapped candidate, against refine_one; frames k = 0, frame_step, ...
    (the emulation thins them to keep the CPU suite short; the GPU run checks every frame)."""
    rep_f, rep_s = StageReport(), StageReport()
    for dd, bd, rd in zip(dec_dumps, base_dumps, ref_dumps):
        cand, score = rd.data
        for i in range(rd.n):
            y = dd.data[i]
            l1, nc = int(rd.l1[i]), int(rd.nc[i])
            _, f0_floor, f0_ceil = rd.groups[int(rd.ugrp[i])]
            base = bd.data[0][i]
            for k in range(0, l1, frame_step):
                for s in range(nc * 7):
                    f = overlapped(base, nc, k, s, l1)
                    gf, gs = cand[i, k, s], score[i, k, s]
                    if not f > 0:
                        assert gf == 0.0 and gs == 0.0
                        continue
                    rf, rs, e_rf, e_rs, ex = refine_one(y, rd.afs, k, f, f0_floor, f0_ceil)
                    if ex:
                        rep_f.excluded += 1
                        continue
                    where = f"utterance {rd.u0 + i} frame {k} slot {s} (f {f:.6f})"
                    assert (gf > 0) == (rf > 0), f"{where}: device {gf}, restatement {rf}"
                    assert abs(gf - rf) <= e_rf, f"{where}: f0 {gf!r} vs {rf!r} (bound {e_rf:.2e})"
                    assert abs(gs - rs) <= e_rs, f"{where}: score {gs!r} vs {rs!r} (bound {e_rs:.2e})"
                    rep_f.compared += 1
                    if rf > 0:
                        rep_f.worst = max(rep_f.worst, abs(gf - rf) / rf)
                        rep_f.worst_bound = max(rep_f.worst_bound, e_rf / rf)
                        rep_s.worst = max(rep_s.worst, abs(gs - rs) / rs)
                        rep_s.worst_bound = max(rep_s.worst_bound, e_rs / rs)
    return rep_f, rep_s


# ------------------------------------------------------------------ cases
def signal(kind, fs, n, seed):
    """the fuzz generator's signal kinds (tests/fuzz/fuzz_emu_parity.py), without digital silence"""
    from synth import synth_batch
    rng = np.random.default_rng(seed)
    x = synth_batch([seed], fs, n).numpy()[0]
    t = np.arange(n) / fs
    if kind == "tone":
        x = 0.3 * np.sin(2 * np.pi * 523.0 * t) + 1e-4 * rng.normal(size=n)
    elif kind == "dc":
        x = x + 0.2
    elif kind == "clipped":
        x = np.clip(x * 8, -1, 1)
    elif kind == "impulses":
        x = np.zeros(n)
        x[::int(fs / 140.0)] = 0.5
        x += 1e-5 * rng.normal(size=n)
    return x


def batch(fs, kinds, lens, seed0=1):
    n = max(lens)
    x = np.zeros((len(lens), n))
    for u, (k, m) in enumerate(zip(kinds, lens)):
        x[u, :m] = signal(k, fs, m, seed0 + u)
    return x


def run_case(world, ref, fs, kinds, lens, ranges, env=None, frame_step=1, last_chunk_only=False):
    """Captures every stage of one batch and checks each against its restatement; returns the per-stage reports."""
    require_extended()
    x = batch(fs, kinds, lens)
    rng = [ranges[u % len(ranges)] for u in range(len(lens))]
    dumps = capture(world, x, fs, rng, lens, env)
    for s in STAGES:
        assert dumps[s], f"no {s} dump written"
    out = {"n_chunks": len(dumps["RAW"])}
    if last_chunk_only:
        dumps = {s: v[-1:] for s, v in dumps.items()}
    out["decimated"] = check_decimated(dumps["DECIMATED"], ref, x, lens)
    out["raw"] = check_raw(dumps["DECIMATED"], dumps["RAW"])
    out["base"] = check_base(dumps["RAW"], dumps["BASE"])
    out["refined"] = check_refined(dumps["DECIMATED"], dumps["BASE"], dumps["REFINED"], frame_step)
    return out


def check_last_chunk(world, ref, frame_step):
    """At the smallest scratch budget (64 MB) a 3 s utterance at 16 kHz sets the strides of the whole batch and
    leaves room for two utterances per chunk: five utterances run in chunks of 2, 2 and 1.  The last chunk, which
    starts at utterance 4 of the batch, is checked."""
    from world_b200.api import World
    small = World(device=world.device, lib_path=world.lib._name, array_module=world.xp)
    try:
        small.set_scratch_budget(64 << 20)
        out = run_case(small, ref, 16000, ["speech", "tone", "speech", "impulses", "clipped"],
                       [48000, 2600, 3200, 2000, 2900], [(71.0, 800.0)], frame_step=frame_step, last_chunk_only=True)
    finally:
        small.close()
    assert out["n_chunks"] == 3
    return out
