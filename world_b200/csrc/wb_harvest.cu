// wb_harvest.cu -- Harvest F0 estimation for a batch (replaces Harvest()/HarvestGeneralBody,
// harvest.cpp:1145-1255).  Algorithm card: SURVEY.md A5.  Everything runs on the 1 ms grid and
// is subsampled to frame_period at the end, exactly like the reference (harvest.cpp:1237-1251).
//   K-HVd  harvest_prep_kernel     edge-padded decimation to ~8 kHz + DC removal      (:43-93)
//   K-HVf  band_sweep_kernel       152 band-pass FIRs + zero-crossing trains + interp1  (:99-343)
//   K-HVp  harvest_detect_kernel   per-frame candidate pooling over channels           (:348-412)
//   K-HVr  harvest_refine_kernel   instantaneous-frequency refinement, one warp per 1 ms frame,
//                                  the +-3 frame overlap (:417-429) done as an index map  (:434-631)
//          harvest_remove_kernel   RemoveUnreliableCandidates                          (:652-688)
//   K-HVc  harvest_contour_kernel  SearchF0Base + FixStep1..4 (sequential per utterance) (:693-1043)
//          harvest_smooth_kernel   zero-lag Butterworth per voiced section + subsample  (:1049-1113, 1246-1251)
// GetMeanF0's two FFTs per candidate are replaced by a sparse DFT at the <= 6 harmonic bins that
// FixF0 reads (same linear functional, SURVEY.md A5 step 5).
#include "wb_internal.h"
#include "wb_f0common.cuh"
#include "wb_spectral.cuh"
#include "wb_mma.cuh"
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

namespace wb {

// Event-list capacity per band and train: crossings of a signal band-limited around/below
// `boundary` cannot be denser than ~boundary per second for long; 2.5x margin, hard bound
// ylen/2+2 (a negative-going crossing needs two samples).  The lists are history rings: more events
// than this wrap around; only a look-back beyond the last `cap` events raises status bit 4.
static void plan_edge_caps(const std::vector<double> &boundary, double afs, int max_ylen, bool full,
                           std::vector<int> *cap, std::vector<long long> *off, size_t *stride) {
  const int nb = (int)boundary.size();
  cap->resize(nb); off->resize(nb);
  long long run = 0;
  long long floor_cap = 2048;
  if (const char *e = getenv("WB_EDGE_CAP_MIN")) floor_cap = atoll(e) > 0 ? atoll(e) : floor_cap;   // test hook: force wraps
  for (int i = 0; i < nb; ++i) {
    const long long hard = (long long)max_ylen / 2 + 2;
    long long soft = (long long)(2.5 * boundary[i] * max_ylen / afs) + 64;
    if (soft < floor_cap) soft = floor_cap;   // a tile can append up to 1025 events per train; the rings look back 256
    // non-decimated input (ripple path): in digital silence the difference trains fire every sample while the
    // crossing trains are silent, so frames cannot be finalised until the silence ends -- keep every event
    if (full) soft = hard;
    (*cap)[i] = (int)(soft < hard ? soft : hard);
    (*off)[i] = run;
    run += 4LL * (*cap)[i];
  }
  *stride = (size_t)run;
}

#define WB_HV_BASE 32        // >= round(channels / 10): base candidates kept per frame
#define WB_HV_WARPS 4

// ------------------------------------------------------------------ K-HVd
struct HvPrepParams {
  const double *x; const int *x_len; int x_stride; int ratio;
  double *y; size_t y_stride; int y_origin; int *y_len;
};

WB_KERNEL(256, 2) harvest_prep_kernel(HvPrepParams p) {
  WB_SHARED double red[WB_RED_DOUBLES];
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int n = p.x_len[u];
  const double *x = p.x + (size_t)u * p.x_stride;
  double *y = p.y + (size_t)u * p.y_stride + p.y_origin;
  const int ylen = static_cast<int>(ceil(static_cast<double>(n) / p.ratio));
  if (p.ratio != 1) {
    // launch_decimate() already wrote the decimated samples (harvest.cpp:43-66)
  } else {
    for (int i = tid; i < n; i += nth) y[i] = x[i];
    WB_SYNC();
  }
  double s = 0.0;
  for (int i = tid; i < ylen; i += nth) s += y[i];
  const double mean = block_sum(s, red) / ylen;
  for (int i = tid; i < ylen; i += nth) y[i] = y[i] - mean;
  if (tid == 0) p.y_len[u] = ylen;
}

// ------------------------------------------------------------------ K-HVp
// Range groups (SweepParams::ugrp): utterance u analyses with group ugrp[u], whose band list has grp_nb channels and
// whose candidates are kept within [grp_floor, grp_ceil].  A uniform batch is one group.
struct HvGroups {
  const int *ugrp; const int *grp_nb; const double *grp_floor, *grp_ceil;
};

struct HvDetectParams {
  const double *raw; int n_bands; int l1_stride; const int *l1;   // raw rows: [n][n_bands = batch maximum][l1_stride]
  HvGroups gr;
  double *base; int *base_count; int *nc;   // [n][l1_stride][WB_HV_BASE], [n][l1_stride], [n]
  int n_utts;
};

WB_KERNEL_PLAIN harvest_detect_kernel(HvDetectParams p) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)p.n_utts * p.l1_stride) return;
  const int u = (int)(g / p.l1_stride), i = (int)(g % p.l1_stride);
  if (i >= p.l1[u]) return;
  const double *raw = p.raw + (size_t)u * p.n_bands * p.l1_stride + i;
  const int nb = p.gr.grp_nb[p.gr.ugrp[u]];
  double *out = p.base + (size_t)g * WB_HV_BASE;
  int count = 0, prev = 0, st = 0;
  double sum = 0.0;
  // vuv[0] = vuv[nb-1] = 0; a section [st, ed) is closed when vuv falls (harvest.cpp:348-385)
  for (int j = 1; j < nb; ++j) {
    const int v = (j == nb - 1) ? 0 : (raw[(size_t)j * p.l1_stride] > 0 ? 1 : 0);
    if (v - prev == 1) { st = j; sum = 0.0; }
    if (v) sum += raw[(size_t)j * p.l1_stride];
    if (v - prev == -1) {
      if (j - st >= 10 && count < WB_HV_BASE) out[count++] = sum / (j - st);
    }
    prev = v;
  }
  for (int c = count; c < WB_HV_BASE; ++c) out[c] = 0.0;
  p.base_count[g] = count;
#ifdef WB_EMU
  if (count > p.nc[u]) p.nc[u] = count;
#else
  if (count > 0) atomicMax(&p.nc[u], count);
#endif
}

// ------------------------------------------------------------------ K-HVr
struct HvRefineParams {
  const double *y; size_t y_stride; int y_origin; const int *y_len; double afs;
  const double *base; const int *nc; int l1_stride; const int *l1; int max_cand;   // max_cand: batch maximum (stride)
  HvGroups gr;                   // the utterance's f0_floor / f0_ceil
  double *cand; double *score;   // [n][l1_stride][max_cand]
  const double2 *tw;
  int nwin_max;
};

#ifdef WB_EMU
#define WB_LANE 0
#define WB_LANES 1
WB_DEV double warp_sum(double v) { return v; }
#else
#define WB_LANE ((int)(threadIdx.x & 31))
#define WB_LANES 32
WB_DEV double warp_sum(double v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif

WB_DEV double2 hv_tw(const double2 *__restrict__ tw, int idx) {
  double2 w = __ldg(&tw[idx & (WB_TW_N / 2 - 1)]);
  if (idx & (WB_TW_N / 2)) { w.x = -w.x; w.y = -w.y; }
  return w;
}

// GetRefinedF0 (harvest.cpp:589-617) for one candidate, executed by one warp.
// wbuf / xbuf / dbuf: per-warp shared scratch of nwin doubles each (window, x*window, x*dwindow).
// Loops are unrolled by four independent iterations per lane to keep several cosines / table
// gathers in flight (the kernel is latency bound otherwise).
// Lane layout of the sparse DFT: lane = 8*c + m handles harmonic m (H <= 6 of the 8 slots) over
// the samples j = c, c+4, c+8, ...; two xor-shuffles fold the four sample classes, then the
// harmonics are combined in index order exactly like FixF0 (harvest.cpp:509-535).
WB_DEV void hv_refine_one(const double *__restrict__ y, int y_len, double afs, double t, double f,
                          double f0_floor, double f0_ceil, const double2 *__restrict__ tw, double *wbuf,
                          double *xbuf, double *dbuf, double *out_f0, double *out_score) {
  const int lane = WB_LANE;
  const int h = static_cast<int>(1.5 * afs / f + 1.0);
  const int nwin = 2 * h + 1;
  int lg = 0;
  while ((2 << lg) <= nwin) ++lg;
  const int lg_nfft = lg + 2, nfft = 1 << lg_nfft;
  const double T = (2.0 * h + 1.0) / afs;
  // base_index[j] = round((t + base_time[0]) * fs + 0.001) + j   (harvest.cpp:434-441)
  const int basic = round_half_away((t + (-h + 0) / afs) * afs + 0.001);
  // Blackman window (harvest.cpp:446-456); cos(2a) = 2 cos(a)^2 - 1 saves the second cosine, and
  // the two per-sample divisions (by afs and by T) become multiplications by reciprocals: the
  // window only has to be accurate to rounding, it feeds no integer decision.
  const double inv_afs = 1.0 / afs, w_scale = 2.0 * kPi / T;
  for (int j0 = 0; j0 < nwin; j0 += 4 * WB_LANES) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + q * WB_LANES + lane;
      if (j < nwin) {
        const double tmp = ((basic + j) - 1.0) * inv_afs - t;
        const double c1 = cos_small(w_scale * tmp);
        wbuf[j] = 0.42 + 0.5 * c1 + 0.08 * (2.0 * c1 * c1 - 1.0);
      }
    }
  }
#ifndef WB_EMU
  __syncwarp();
#endif
  for (int j0 = 0; j0 < nwin; j0 += 4 * WB_LANES) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + q * WB_LANES + lane;
      if (j < nwin) {
        double dw;
        if (j == 0) dw = -wbuf[1] / 2.0;
        else if (j == nwin - 1) dw = wbuf[nwin - 2] / 2.0;
        else dw = -(wbuf[j + 1] - wbuf[j - 1]) / 2.0;
        const double s = y[imax(0, imin(y_len - 1, basic + j - 1))];
        xbuf[j] = s * wbuf[j];
        dbuf[j] = s * dw;
      }
    }
  }
#ifndef WB_EMU
  __syncwarp();
#endif
  const int H = imin(static_cast<int>(afs / 2.0 / f), 6);
  const int shift = WB_TW_LOG2 - lg_nfft;
  double amp_l = 0.0, inst_l = 0.0;
  double numerator = 0.0, denominator = 0.0, score = 0.0;
#ifdef WB_EMU
  for (int m = 0; m < H; ++m) {
    const int c0 = 0, cstep = 1;
#else
  {
    const int m = lane & 7, c0 = lane >> 3, cstep = 4;
#endif
    double mr = 0.0, mi = 0.0, dr = 0.0, di = 0.0;
    const int bin = round_half_away(f * nfft / afs * (m + 1));
    if (m < H) {
      // twiddles exp(-j 2 pi bin j / nfft) by rotation: four interleaved chains (one per unrolled
      // slot) start from exact table values and advance by exp(-j 2 pi bin 4 cstep / nfft); a
      // chain is <= nwin / (4 cstep) steps long, so the accumulated rounding stays ~1e-15.
      // (A table gather per sample made this kernel L1-LSU bound.)
      const double2 rot = hv_tw(tw, ((bin * 4 * cstep) & (nfft - 1)) << shift);
      double2 wq[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) wq[q] = hv_tw(tw, ((bin * (c0 + q * cstep)) & (nfft - 1)) << shift);
      for (int j0 = c0; j0 < nwin; j0 += 4 * cstep) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int j = j0 + q * cstep;
          if (j < nwin) {
            const double2 w = wq[q];
            const double a = xbuf[j], d = dbuf[j];
            mr = fma(a, w.x, mr); mi = fma(a, w.y, mi);
            dr = fma(d, w.x, dr); di = fma(d, w.y, di);
          }
          const double nx = fma(wq[q].x, rot.x, -(wq[q].y * rot.y));
          const double ny = fma(wq[q].x, rot.y, wq[q].y * rot.x);
          wq[q].x = nx; wq[q].y = ny;
        }
      }
    }
#ifndef WB_EMU
    mr += __shfl_xor_sync(0xffffffffu, mr, 8);  mi += __shfl_xor_sync(0xffffffffu, mi, 8);
    dr += __shfl_xor_sync(0xffffffffu, dr, 8);  di += __shfl_xor_sync(0xffffffffu, di, 8);
    mr += __shfl_xor_sync(0xffffffffu, mr, 16); mi += __shfl_xor_sync(0xffffffffu, mi, 16);
    dr += __shfl_xor_sync(0xffffffffu, dr, 16); di += __shfl_xor_sync(0xffffffffu, di, 16);
#endif
    const double num = mr * di - mi * dr;
    const double pw = mr * mr + mi * mi;
    inst_l = pw == 0.0 ? 0.0 : static_cast<double>(bin) * afs / nfft + num / pw * afs / 2.0 / kPi;
    amp_l = sqrt(pw);
    // this harmonic's three FixF0 terms (harvest.cpp:521-527); summed in harmonic order below
    const double t_num = amp_l * inst_l;
    const double t_den = amp_l * (m + 1.0);
    const double t_sc = fabs((inst_l / (m + 1.0) - f) / f);
#ifdef WB_EMU
    numerator += t_num;
    denominator += t_den;
    score += t_sc;
  }
#else
    for (int mm = 0; mm < H; ++mm) {
      numerator += __shfl_sync(0xffffffffu, t_num, mm);
      denominator += __shfl_sync(0xffffffffu, t_den, mm);
      score += __shfl_sync(0xffffffffu, t_sc, mm);
    }
  }
#endif
  double rf = numerator / (denominator + kTiny);
  double rs = 1.0 / (score / H + kTiny);
  if (rf < f0_floor || rf > f0_ceil || rs < 2.5) { rf = 0.0; rs = 0.0; }
  *out_f0 = rf;
  *out_score = rs;
#ifndef WB_EMU
  __syncwarp();
#endif
}

// candidate of overlapped slot s at frame k (OverlapF0Candidates, harvest.cpp:417-429)
WB_DEV double hv_slot_candidate(const double *__restrict__ base, int L1, int nc, int k, int s) {
  const int grp = s / nc, j = s % nc;
  int src = k;
  if (grp >= 1 && grp <= 3) src = k - grp;
  else if (grp >= 4) src = k + (grp - 3);
  if (src < 0 || src >= L1 || j >= WB_HV_BASE) return 0.0;
  return base[(size_t)src * WB_HV_BASE + j];
}

WB_KERNEL(32 * WB_HV_WARPS, 6) harvest_refine_kernel(HvRefineParams p) {
  WB_DYN_SMEM(double, smem);
#ifdef WB_EMU
  const int warp = 0, nwarps = 1;
#else
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#endif
  const int lane = WB_LANE;
  const int u = blockIdx.y;
  const int L1 = p.l1[u];
  const int k = blockIdx.x * nwarps + warp;
  if (k >= L1) return;
  const int nc = p.nc[u], n_slots = nc * 7;
  double *wbuf = smem + (size_t)warp * 3 * p.nwin_max, *xbuf = wbuf + p.nwin_max, *dbuf = xbuf + p.nwin_max;
  const double *y = p.y + (size_t)u * p.y_stride + p.y_origin;
  const double *base = p.base + (size_t)u * p.l1_stride * WB_HV_BASE;
  double *cand = p.cand + ((size_t)u * p.l1_stride + k) * p.max_cand;
  double *score = p.score + ((size_t)u * p.l1_stride + k) * p.max_cand;
  const double t = k * 1 / 1000.0;  // basic frame period 1 ms (harvest.cpp:1203)
  const int y_len = p.y_len[u];
  const int grp = p.gr.ugrp[u];
  const double f0_floor = p.gr.grp_floor[grp], f0_ceil = p.gr.grp_ceil[grp];
  // the frame's slots are fetched WB_LANES at a time (one per lane) and handed round by shuffle
  for (int s0 = 0; s0 < n_slots; s0 += WB_LANES) {
    const double f_mine = (s0 + lane < n_slots) ? hv_slot_candidate(base, L1, nc, k, s0 + lane) : 0.0;
    double rf_mine = 0.0, rs_mine = 0.0;
    for (int q = 0; q < WB_LANES && s0 + q < n_slots; ++q) {
#ifdef WB_EMU
      const double f = f_mine;
#else
      const double f = __shfl_sync(0xffffffffu, f_mine, q);
#endif
      if (f > 0.0) {
        double rf, rs;
        hv_refine_one(y, y_len, p.afs, t, f, f0_floor, f0_ceil, p.tw, wbuf, xbuf, dbuf, &rf, &rs);
        if (lane == q) { rf_mine = rf; rs_mine = rs; }
      }
    }
    if (s0 + lane < n_slots) { cand[s0 + lane] = rf_mine; score[s0 + lane] = rs_mine; }
  }
}

// ------------------------------------------------------------------ K-HVr, chain variant (the default where it applies)
// DESIGN.md 9 item 2.  When one 1 ms frame is a whole number S of decimated samples (8000 Hz: S = 8), the
// seven overlapped refinements of a base candidate (frames k-3 .. k+3) share one window and one set of
// twiddles: GetBaseIndex gives basic = S k' - h, so the window argument (basic + i - 1) / afs - t_k' is
// (i - h - 1) / afs for every frame.  One warp per SOURCE frame k loops over its base candidates.  Outputs go to
// slot j of frame k, slot j + nc g of frame k + g and slot j + nc (g + 3) of frame k - g (the inverse of
// hv_slot_candidate); every other slot keeps the zero the driver memset.
// Default wherever S is integral (the per-frame kernel recomputes each template seven times; f0 stays within the
// parity bound with no V/UV flip); WB_NO_REFINE_CHAIN=1 selects the per-frame kernel for A/B runs.
//
// The seven sparse DFTs of a candidate are one matrix product on the FP64 tensor cores, C = T X:
//  * T (A operand, two 16-row tiles): tile 0 rows m / m + 8 = w[i] cos / sin of harmonic m's twiddle at sample i,
//    tile 1 the same with dw; rows of harmonics m >= H are zero.
//  * X (B operand): X[i][g] = x[i + S g], the sample under window position i in frame k + g - 3 (column 7 is
//    computed and discarded).
//  * k order inside a k-step q: slot t carries sample 8 q + 2 t and slot t + 4 sample 8 q + 2 t + 1, so a lane's
//    window values come from one row of the window table and its two twiddles advance by e^{-j theta_m 8} per step.
// The C fragments leave lane (m, t) holding {main re, main im, diff re, diff im} of harmonic m for frames 2t and
// 2t + 1; FixF0 sums the harmonics in index order by shuffle.

// The window (harvest.cpp:446-456) and its derivative depend on h only.  Row h of the window table starts at
// hv_win_offset(h) doubles and holds, for k-step q and slot t, {w[8q+2t], w[8q+2t+1], dw[8q+2t], dw[8q+2t+1]} at
// 4 (4 q + t): two 16-byte loads per lane and step.  The row has 8 ceil(nwin / 8) samples, zero from nwin on.
WB_HD inline int hv_win_offset(int h) {   // 16 sum_{h' < h} (h' / 4 + 1)
  const int a = h >> 2, b = h & 3;
  return 16 * (h + 2 * a * (a - 1) + a * b);
}

WB_DEV double hv_window(int i, int h, double afs) {
  const double T = (2.0 * h + 1.0) / afs;
  const double inv_afs = 1.0 / afs, w_scale = 2.0 * kPi / T;
  const double tau = (i - h - 1.0) * inv_afs;
  const double c1 = cos_small(w_scale * tau);
  return 0.42 + 0.5 * c1 + 0.08 * (2.0 * c1 * c1 - 1.0);
}

struct HvWindowParams {
  double *win; double afs;
};

// block h: row h of the window table
WB_KERNEL_PLAIN harvest_window_table_kernel(HvWindowParams p) {
  const int h = blockIdx.x, nwin = 2 * h + 1, len = 8 * ((nwin + 7) >> 3);
  double *row = p.win + hv_win_offset(h);
  for (int i = WB_TID; i < len; i += WB_NTH) {
    double w = 0.0, dw = 0.0;
    if (i < nwin) {
      w = hv_window(i, h, p.afs);
      if (i == 0) dw = -hv_window(1, h, p.afs) / 2.0;
      else if (i == nwin - 1) dw = hv_window(nwin - 2, h, p.afs) / 2.0;
      else dw = -(hv_window(i + 1, h, p.afs) - hv_window(i - 1, h, p.afs)) / 2.0;
    }
    const int o = 4 * (4 * (i >> 3) + ((i & 7) >> 1)) + (i & 1);
    row[o] = w;
    row[o + 2] = dw;
  }
}

// element `src` of a per-lane value, read by every lane at once (src may differ per lane); on the host the
// array must have been filled by an earlier WB_FOR_LANES block
#ifdef WB_EMU
#define WB_LANE_READ(arr, src) (arr[(src)])
#else
#define WB_LANE_READ(arr, src) __shfl_sync(0xffffffffu, arr[0], (src))
#endif

struct HvChainParams {
  HvRefineParams r;
  int frame_samples;   // S
  const double *win;   // window table, rows h = 0 .. nwin_max / 2
};

// doubles of one warp's signal segment: the window at h = nwin_max / 2 padded to whole k-steps, read up to 7 S later
// for column 7 (an even count keeps every warp's segment 16-byte aligned)
WB_HD inline int hv_chain_seg(int nwin_max, int S) { return ((nwin_max / 2) * 2 + 8 + 7 * S + 1) & ~1; }

WB_DEV void refine_chain_body(const HvChainParams &cp) {
  WB_DYN_SMEM(double, smem);
  const HvRefineParams &p = cp.r;
#ifdef WB_EMU
  const int warp = 0, nwarps = 1;
#else
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#endif
  const int u = blockIdx.y;
  const int L1 = p.l1[u];
  const int k = blockIdx.x * nwarps + warp;   // source frame
  if (k >= L1) return;
  const int S = cp.frame_samples;
  const int nc = p.nc[u];
  const int grp = p.gr.ugrp[u];
  const double f0_floor = p.gr.grp_floor[grp], f0_ceil = p.gr.grp_ceil[grp];
  const int hs = p.nwin_max / 2;   // the largest h the window table and the segment serve (the batch's lowest floor)
  const int seg = hv_chain_seg(p.nwin_max, S);
  double *xs = smem + (size_t)warp * seg;
  const double *y = p.y + (size_t)u * p.y_stride + p.y_origin;
  const int y_len = p.y_len[u];
  const double afs = p.afs;
  const double *base = p.base + ((size_t)u * p.l1_stride + k) * WB_HV_BASE;
  // signal of frames k-3 .. k+4 under the window at h = hs: a candidate with h <= hs reads it from hs - h on
  WB_FOR_LANES(l) {
    const int basic0 = S * (k - 3) - hs;
    for (int i = l; i < seg; i += 32) xs[i] = y[imax(0, imin(y_len - 1, basic0 + i - 1))];
  }
#ifndef WB_EMU
  __syncwarp();
#endif
  for (int j = 0; j < nc && j < WB_HV_BASE; ++j) {
    const double f = base[j];
    if (!(f > 0.0)) continue;
    const int h = static_cast<int>(1.5 * afs / f + 1.0);
    if (h > hs) continue;   // nwin_max covers f >= the lowest f0_floor of the batch
    const int nwin = 2 * h + 1;
    int lg = 0;
    while ((2 << lg) <= nwin) ++lg;
    const int lg_nfft = lg + 2, nfft = 1 << lg_nfft;
    const int H = imin(static_cast<int>(afs / 2.0 / f), 6);
    const int shift = WB_TW_LOG2 - lg_nfft;
    const int nq = (nwin + 7) >> 3;
    const double *xc = xs + (hs - h);
    const double2 *wt = reinterpret_cast<const double2 *>(cp.win + hv_win_offset(h));
    double cw[WB_CL][4], cd[WB_CL][4];   // C fragments of the w tile and the dw tile
    double2 e0[WB_CL], e1[WB_CL], rot[WB_CL];
    WB_FOR_LANES(l) {
      const int m = l >> 2, t = l & 3;
#pragma unroll
      for (int e = 0; e < 4; ++e) { cw[WB_LI(l)][e] = 0.0; cd[WB_LI(l)][e] = 0.0; }
      e0[WB_LI(l)] = e1[WB_LI(l)] = rot[WB_LI(l)] = make_double2(0.0, 0.0);
      if (m < H) {
        // twiddles exp(-j 2 pi bin i / nfft) of samples 2t and 2t + 1 by rotation from exact table values; a chain
        // is nwin / 8 steps long, so the accumulated rounding stays ~1e-15
        const int bin = round_half_away(f * nfft / afs * (m + 1));
        rot[WB_LI(l)] = hv_tw(p.tw, ((bin * 8) & (nfft - 1)) << shift);
        e0[WB_LI(l)] = hv_tw(p.tw, ((bin * 2 * t) & (nfft - 1)) << shift);
        e1[WB_LI(l)] = hv_tw(p.tw, ((bin * (2 * t + 1)) & (nfft - 1)) << shift);
      }
    }
    for (int q = 0; q < nq; ++q) {
      double aw[WB_CL][4], ad[WB_CL][4], bx[WB_CL][2];
      WB_FOR_LANES(l) {
        const int g = l >> 2, t = l & 3;
        const double2 w = __ldg(&wt[2 * (4 * q + t)]), dw = __ldg(&wt[2 * (4 * q + t) + 1]);
        double2 &a = e0[WB_LI(l)], &b = e1[WB_LI(l)];
        const double2 r = rot[WB_LI(l)];
        aw[WB_LI(l)][0] = w.x * a.x;  aw[WB_LI(l)][1] = w.x * a.y;  aw[WB_LI(l)][2] = w.y * b.x;  aw[WB_LI(l)][3] = w.y * b.y;
        ad[WB_LI(l)][0] = dw.x * a.x; ad[WB_LI(l)][1] = dw.x * a.y; ad[WB_LI(l)][2] = dw.y * b.x; ad[WB_LI(l)][3] = dw.y * b.y;
        const int xi = 8 * q + 2 * t + S * g;
        bx[WB_LI(l)][0] = xc[xi];
        bx[WB_LI(l)][1] = xc[xi + 1];
        const double ax = fma(a.x, r.x, -(a.y * r.y)), ay = fma(a.x, r.y, a.y * r.x);
        const double bxx = fma(b.x, r.x, -(b.y * r.y)), by = fma(b.x, r.y, b.y * r.x);
        a.x = ax; a.y = ay; b.x = bxx; b.y = by;
      }
      mma_f64_16x8x8(cw, aw, bx);
      mma_f64_16x8x8(cd, ad, bx);
    }
    // FixF0 (harvest.cpp:498-535): each lane's harmonic terms for frames 2t and 2t + 1, then the sums over the
    // harmonics in index order (lanes 4 mm + t), written by lanes 0-3
    double t_num[2][WB_CL], t_den[2][WB_CL], t_sc[2][WB_CL];
    WB_FOR_LANES(l) {
      const int m = l >> 2;
      const int bin = round_half_away(f * nfft / afs * (m + 1));
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const double mr = cw[WB_LI(l)][e], mi = cw[WB_LI(l)][2 + e], dr = cd[WB_LI(l)][e], di = cd[WB_LI(l)][2 + e];
        const double num = mr * di - mi * dr;
        const double pw = mr * mr + mi * mi;
        const double inst = pw == 0.0 ? 0.0 : static_cast<double>(bin) * afs / nfft + num / pw * afs / 2.0 / kPi;
        const double amp = sqrt(pw);
        t_num[e][WB_LI(l)] = amp * inst;
        t_den[e][WB_LI(l)] = amp * (m + 1.0);
        t_sc[e][WB_LI(l)] = fabs((inst / (m + 1.0) - f) / f);
      }
    }
    WB_FOR_LANES(l) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int g = 2 * (l & 3) + e, kk = k + g - 3;
        double numerator = 0.0, denominator = 0.0, score = 0.0;
        for (int mm = 0; mm < H; ++mm) {
          const int src = 4 * mm + (l & 3);
          numerator += WB_LANE_READ(t_num[e], src);
          denominator += WB_LANE_READ(t_den[e], src);
          score += WB_LANE_READ(t_sc[e], src);
        }
        if (l < 4 && g < 7 && kk >= 0 && kk < L1) {
          double rf = numerator / (denominator + kTiny);
          double rs = 1.0 / (score / H + kTiny);
          if (rf < f0_floor || rf > f0_ceil || rs < 2.5) { rf = 0.0; rs = 0.0; }
          const int d = g - 3;
          const int slot = d == 0 ? j : (d > 0 ? j + nc * d : j + nc * (3 - d));
          p.cand[((size_t)u * p.l1_stride + kk) * p.max_cand + slot] = rf;
          p.score[((size_t)u * p.l1_stride + kk) * p.max_cand + slot] = rs;
        }
      }
    }
  }
}

// 8 CTAs per SM (64 registers, a few spills around the MMA loop) beat 6 (80 registers) and 5 (96, no spills) on H100
WB_KERNEL(32 * WB_HV_WARPS, 8) harvest_refine_chain_kernel(HvChainParams cp) { refine_chain_body(cp); }

// ------------------------------------------------------------------ RemoveUnreliableCandidates
struct HvRemoveParams {
  const double *cand_in; const double *score_in; double *cand; double *score;
  const int *nc; const int *l1; int l1_stride; int max_cand; int n_utts;
  double *f0_base;   // [n][5][l1_stride] work rows of the contour kernel; row 0 = SearchF0Base result
};

// min(1, min_c |reference - row[c]| / reference): SelectBestF0's error with allowed_range 1.0
// (harvest.cpp:657-661).  Division by the positive reference is monotone under rounding, so the
// minimum of the quotients is the quotient of the minimum: one division per call.
WB_DEV double hv_min_rel_error(double reference, const double *row, int n) {
  double dmin_abs = fabs(reference - row[0]);
  for (int c = 1; c < n; ++c) dmin_abs = dmin(dmin_abs, fabs(reference - row[c]));
  const double e = dmin_abs / reference;
  return e > 1.0 ? 1.0 : e;
}

// One warp per 1 ms frame, lanes over the frame's candidate slots (round 1 ran one THREAD per frame: rows of 105
// doubles read with an 840-byte stride between threads; 40 ms per 1024 x 10 s).  Neighbour rows are read by all
// lanes at the same address (broadcast).  SearchF0Base keeps the FIRST slot with the highest score: the warp
// arg-max breaks ties towards the lower slot index.
#define WB_RM_WARPS 8
WB_KERNEL(32 * WB_RM_WARPS, 4) harvest_remove_kernel(HvRemoveParams p) {
#ifdef WB_EMU
  const int warp = 0, nwarps = 1;
#else
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#endif
  const int lane = WB_LANE;
  const long long g = (long long)blockIdx.x * nwarps + warp;
  if (g >= (long long)p.n_utts * p.l1_stride) return;
  const int u = (int)(g / p.l1_stride), i = (int)(g % p.l1_stride);
  const int L1 = p.l1[u];
  if (i >= L1) return;
  const int n = p.nc[u] * 7;
  const double *row = p.cand_in + (size_t)g * p.max_cand;
  double *oc = p.cand + (size_t)g * p.max_cand, *os = p.score + (size_t)g * p.max_cand;
  const double *srow = p.score_in + (size_t)g * p.max_cand;
  const bool interior = i >= 1 && i < L1 - 1;
  double best = 0.0, best_score = 0.0;  // SearchF0Base (harvest.cpp:693-705) on the cleaned candidates
  int best_j = 0x7fffffff;
  for (int j = lane; j < n; j += WB_LANES) {
    double c = row[j], s = srow[j];
    if (interior && c != 0) {
      const double e1 = hv_min_rel_error(c, row + p.max_cand, n);
      const double e2 = hv_min_rel_error(c, row - p.max_cand, n);
      if (dmin(e1, e2) > 0.05) { c = 0.0; s = 0.0; }
    }
    oc[j] = c; os[j] = s;
    if (s > best_score) { best = c; best_score = s; best_j = j; }
  }
#ifndef WB_EMU
  for (int o = 16; o; o >>= 1) {
    const double s2 = __shfl_xor_sync(0xffffffffu, best_score, o);
    const double c2 = __shfl_xor_sync(0xffffffffu, best, o);
    const int j2 = __shfl_xor_sync(0xffffffffu, best_j, o);
    if (s2 > best_score || (s2 == best_score && j2 < best_j)) { best_score = s2; best = c2; best_j = j2; }
  }
#endif
  if (lane == 0) p.f0_base[(size_t)u * 5 * p.l1_stride + i] = best;
}

// ------------------------------------------------------------------ K-HVc
struct HvContourParams {
  const double *cand; const double *score; const int *nc; const int *l1; int l1_stride; int max_cand;
  double *work;      // [n][5][l1_stride]: base, s1, s2, s3, s4
  int *iwork;        // [n][6][l1_stride]: boundary list, section descriptors (off, lo, hi), order
  double *mc;        // [n][mc_stride] sparse multi-channel storage
  size_t mc_stride;
  int *status;
};

// GetBoundaryList (harvest.cpp:727-743), block-cooperative: every thread scans a contiguous
// chunk, chunk counts are prefix-summed, boundaries are written in order.  list[k] = i - k % 2.
// `cnt` is shared scratch of nthreads + 1 ints.  Returns the number of boundaries to all threads.
WB_DEV int hv_boundaries(const double *f0, int n, int *list, int *cnt) {
  const int tid = WB_TID, nth = WB_NTH;
  const int chunk = (n - 1 + nth - 1) / nth;  // positions 1 .. n-1
  const int lo = imin(n, 1 + tid * chunk), hi = imin(n, lo + chunk);
  int c = 0;
  for (int i = lo; i < hi; ++i) {
    const int v = (i == n - 1) ? 0 : (f0[i] > 0 ? 1 : 0);
    const int pv = (i - 1 == 0) ? 0 : (f0[i - 1] > 0 ? 1 : 0);
    c += (v != pv);
  }
  WB_SYNC();
  cnt[tid] = c;
  WB_SYNC();
  if (tid == 0) {
    int run = 0;
    for (int t = 0; t < nth; ++t) { const int v = cnt[t]; cnt[t] = run; run += v; }
    cnt[nth] = run;
  }
  WB_SYNC();
  int k = cnt[tid];
  for (int i = lo; i < hi; ++i) {
    const int v = (i == n - 1) ? 0 : (f0[i] > 0 ? 1 : 0);
    const int pv = (i - 1 == 0) ? 0 : (f0[i - 1] > 0 ? 1 : 0);
    if (v != pv) { list[k] = i - k % 2; ++k; }
  }
  const int total = cnt[nth];
  WB_SYNC();
  return total;
}

// SelectBestF0 (harvest.cpp:636-650): last candidate among those with the smallest error <= allowed
WB_DEV double hv_select_best(double reference, const double *row, int n, double allowed) {
  double best = 0.0, best_err = allowed;
  for (int c = 0; c < n; ++c) {
    const double e = fabs(reference - row[c]) / reference;
    if (e > best_err) continue;
    best = row[c];
    best_err = e;
  }
  return best;
}

// ExtendF0 (harvest.cpp:791-822) on one section's window `w` (w[j - lo] = contour at frame j)
WB_DEV int hv_extend(double *w, int lo, int hi, int origin, int last_point, int shift, const double *cand,
                     int max_cand, int n_cand, double allowed) {
  const int threshold = 4;
  double tmp_f0 = w[origin - lo];
  int shifted_origin = origin;
  const int distance = last_point > origin ? last_point - origin : origin - last_point;
  int count = 0;
  for (int i = 0; i <= distance; ++i) {
    const int target = origin + shift * i + shift;
    const double v = hv_select_best(tmp_f0, cand + (size_t)target * max_cand, n_cand, allowed);
    if (target >= lo && target <= hi) w[target - lo] = v;
    if (v == 0.0) {
      ++count;
    } else {
      tmp_f0 = v;
      count = 0;
      shifted_origin = target;
    }
    if (count == threshold) break;
  }
  return shifted_origin;
}

WB_DEV double hv_search_score(double f0, const double *crow, const double *srow, int n) {
  double score = 0.0;
  for (int i = 0; i < n; ++i)
    if (f0 == crow[i] && score < srow[i]) score = srow[i];
  return score;
}

WB_KERNEL(128, 4) harvest_contour_kernel(HvContourParams p) {
  WB_SHARED int cnt[130];
  WB_SHARED int sh_nch;
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int L = p.l1[u], nc7 = p.nc[u] * 7, mcand = p.max_cand;
  const double *cand = p.cand + (size_t)u * p.l1_stride * mcand;
  const double *score = p.score + (size_t)u * p.l1_stride * mcand;
  double *fb = p.work + (size_t)u * 5 * p.l1_stride, *s1 = fb + p.l1_stride, *s2 = s1 + p.l1_stride;
  double *s3 = s2 + p.l1_stride, *s4 = s3 + p.l1_stride;
  int *bl = p.iwork + (size_t)u * 6 * p.l1_stride;
  double *mc = p.mc + (size_t)u * p.mc_stride;
  int *off = bl + p.l1_stride, *wlo = off + p.l1_stride, *whi = wlo + p.l1_stride, *order = whi + p.l1_stride;

  // SearchF0Base (:693-705) was evaluated by harvest_remove_kernel while it held the rows: fb[]
  // FixStep1 (:710-722), allowed_range 0.008
  for (int i = tid; i < L; i += nth) {
    double v = 0.0;
    if (i >= 2 && fb[i] != 0.0) {
      const double reference = fb[i - 1] * 2 - fb[i - 2];
      v = (fabs((fb[i] - reference) / reference) > 0.008 && fabs((fb[i] - fb[i - 1])) / fb[i - 1] > 0.008) ? 0.0 : fb[i];
    }
    s1[i] = v;
    s2[i] = v;
  }
  WB_SYNC();
  // FixStep2 (:748-762): voiced sections shorter than 6 frames are removed
  int nb = hv_boundaries(s1, L, bl, cnt);
  for (int i = tid; i < nb / 2; i += nth) {
    if (bl[i * 2 + 1] - bl[i * 2] >= 6) continue;
    for (int j = bl[i * 2]; j <= bl[i * 2 + 1]; ++j) s2[j] = 0.0;
  }
  WB_SYNC();

  // FixStep3 (:978-995): extend sections, select, merge
  for (int i = tid; i < L; i += nth) s3[i] = s2[i];
  nb = hv_boundaries(s2, L, bl, cnt);
  const int nsec = nb / 2;
  if (tid == 0) {
    size_t used = 0;
    int okay = 1;
    for (int s = 0; s < nsec; ++s) {
      const int lo = imax(0, bl[2 * s] - 104), hi = imin(L - 1, bl[2 * s + 1] + 104);
      if (used + (size_t)(hi - lo + 1) > p.mc_stride) { okay = 0; break; }
      off[s] = (int)used; wlo[s] = lo; whi[s] = hi;
      used += (size_t)(hi - lo + 1);
    }
    sh_nch = okay ? 0 : -1;
    if (!okay) atomicOr_status(p.status, 4);
  }
  WB_SYNC();
  if (sh_nch < 0) return;
  // sections are independent until ExtendSub: one thread per section fills its window and runs
  // both ExtendF0 calls (Extend, :858-874)
  for (int s = tid; s < nsec; s += nth) {
    const int st = bl[2 * s], ed = bl[2 * s + 1], lo = wlo[s], hi = whi[s];
    double *w = mc + off[s];
    for (int j = lo; j <= hi; ++j) w[j - lo] = (j >= st && j <= ed) ? s2[j] : 0.0;
    const int new_ed = hv_extend(w, lo, hi, ed, imin(L - 2, ed + 100), 1, cand, mcand, nc7, 0.18);
    const int new_st = hv_extend(w, lo, hi, st, imax(1, st - 100), -1, cand, mcand, nc7, 0.18);
    bl[2 * s + 1] = new_ed;
    bl[2 * s] = new_st;
  }
  WB_SYNC();
  if (tid == 0) {
    // ExtendSub (:839-856): note mean_f0 is NOT reset between sections in the reference
    int nch = 0;
    double mean_f0 = 0.0;
    for (int s = 0; s < nsec; ++s) {
      const int st = bl[2 * s], ed = bl[2 * s + 1];
      const double *w = mc + off[s] - wlo[s];
      for (int j = st; j < ed; ++j) mean_f0 += w[j];
      mean_f0 /= ed - st;
      if (2200.0 / mean_f0 < ed - st) {
        int t;  // Swap(count, s): contour and boundary pair
        t = off[nch]; off[nch] = off[s]; off[s] = t;
        t = wlo[nch]; wlo[nch] = wlo[s]; wlo[s] = t;
        t = whi[nch]; whi[nch] = whi[s]; whi[s] = t;
        t = bl[2 * nch]; bl[2 * nch] = bl[2 * s]; bl[2 * s] = t;
        t = bl[2 * nch + 1]; bl[2 * nch + 1] = bl[2 * s + 1]; bl[2 * s + 1] = t;
        ++nch;
      }
    }
    sh_nch = nch;
  }
  WB_SYNC();
  const int nch = sh_nch;
  if (nch != 0) {
    // MergeF0 (:941-973); merged starts as channel 0 over the whole axis
    {
      const int lo = wlo[0], hi = whi[0];
      const double *w = mc + off[0] - lo;
      for (int i = tid; i < L; i += nth) s3[i] = (i < lo || i > hi) ? 0.0 : w[i];
    }
    WB_SYNC();
    if (tid == 0) {
      for (int i = 0; i < nch; ++i) order[i] = i;
      // MakeSortedOrder exactly as written in the reference (:881-893): the inner loop keeps
      // comparing against position i while elements move
      for (int i = 1; i < nch; ++i)
        for (int j = i - 1; j >= 0; --j) {
          if (bl[order[j] * 2] > bl[order[i] * 2]) { const int t = order[i]; order[i] = order[j]; order[j] = t; }
          else break;
        }
      for (int i = 1; i < nch; ++i) {
        const int o = order[i];
        const int lo = wlo[o], hi = whi[o];
        const double *w = mc + off[o] - lo;
#define WB_CH(j) (((j) < lo || (j) > hi) ? 0.0 : w[(j)])
        if (bl[o * 2] - bl[1] > 0) {
          for (int j = bl[o * 2]; j <= bl[o * 2 + 1]; ++j) s3[j] = WB_CH(j);
          bl[0] = bl[o * 2];
          bl[1] = bl[o * 2 + 1];
        } else {
          // MergeF0Sub (:912-935)
          const int st1 = bl[0], ed1 = bl[1], st2 = bl[o * 2], ed2 = bl[o * 2 + 1];
          if (st1 <= st2 && ed1 >= ed2) {
            bl[1] = ed1;
          } else {
            double score1 = 0.0, score2 = 0.0;
            for (int k = st2; k <= ed1; ++k) {
              score1 += hv_search_score(s3[k], cand + (size_t)k * mcand, score + (size_t)k * mcand, nc7);
              score2 += hv_search_score(WB_CH(k), cand + (size_t)k * mcand, score + (size_t)k * mcand, nc7);
            }
            if (score1 > score2) { for (int k = ed1; k <= ed2; ++k) s3[k] = WB_CH(k); }
            else { for (int k = st2; k <= ed2; ++k) s3[k] = WB_CH(k); }
            bl[1] = ed2;
          }
        }
#undef WB_CH
      }
    }
    WB_SYNC();
  }
  // FixStep4 (:1000-1022): bridge gaps shorter than 9 frames
  for (int i = tid; i < L; i += nth) s4[i] = s3[i];
  nb = hv_boundaries(s3, L, bl, cnt);
  for (int i = tid; i < nb / 2 - 1; i += nth) {
    const int distance = bl[(i + 1) * 2] - bl[i * 2 + 1] - 1;
    if (distance >= 9) continue;
    const double tmp0 = s3[bl[i * 2 + 1]] + 1;
    const double tmp1 = s3[bl[(i + 1) * 2]] - 1;
    const double coefficient = (tmp1 - tmp0) / (distance + 1.0);
    int count = 1;
    for (int j = bl[i * 2 + 1] + 1; j <= bl[(i + 1) * 2] - 1; ++j) s4[j] = tmp0 + coefficient * count++;
  }
}

// ------------------------------------------------------------------ smoothing + subsampling
struct HvSmoothParams {
  const double *work; int l1_stride; const int *l1;  // s4 = work[u][4]
  double *padded;      // [n][pad_stride]: f0 contour padded by 300 zeros on both sides
  double *tmp;         // [n][sec_slots][seg_cap] per-thread section scratch
  int *blist;          // [n][pad_stride]
  double *basic;       // [n][l1_stride] smoothed 1 ms contour
  size_t pad_stride; int sec_slots; int seg_cap;
  const int *f_len; int f_stride; double frame_period;
  double *time_axis; double *f0;
};

// FilteringF0 (harvest.cpp:1049-1074) for one section.  The reference filters the whole padded
// contour (edge-held outside [st, ed]) forward and backward from zero state.  The filter's poles
// have |z| = 0.875, so a zero-state start WB_HV_RUNIN samples before the section is
// indistinguishable (0.875^640 < 1e-37) from the reference's start at sample 0; both passes are
// restricted to [st - RUNIN, ed + RUNIN].  tmp_x holds the reversed forward output of that span.
#define WB_HV_RUNIN 640
WB_DEV void hv_filter_section(const double *f0c, int len, int st, int ed, double *tmp_x, double *basic, int lag) {
  const double b0 = 0.0078202080334971724, b1 = 0.015640416066994345;
  const double a0 = 1.7347257688092754, a1 = -0.76600660094326412;
  const int lo = imax(0, st - WB_HV_RUNIN), hi = imin(len - 1, ed + WB_HV_RUNIN);
  double w0 = 0.0, w1 = 0.0;
  for (int i = lo; i <= hi; ++i) {
    const double xi = f0c[i < st ? st : (i > ed ? ed : i)];
    const double wt = xi + a0 * w0 + a1 * w1;
    tmp_x[hi - i] = b0 * wt + b1 * w0 + b0 * w1;
    w1 = w0; w0 = wt;
  }
  w0 = w1 = 0.0;
  for (int i = 0; i <= hi - lo; ++i) {
    const double wt = tmp_x[i] + a0 * w0 + a1 * w1;
    const int o = hi - i;
    if (o >= st && o <= ed) basic[o - lag] = b0 * wt + b1 * w0 + b0 * w1;
    w1 = w0; w0 = wt;
  }
}

WB_KERNEL(128, 4) harvest_smooth_kernel(HvSmoothParams p) {
  WB_SHARED int cnt[130];
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int L = p.l1[u], lag = 300, len = L + 2 * lag;
  const double *s4 = p.work + ((size_t)u * 5 + 4) * p.l1_stride;
  double *pad = p.padded + (size_t)u * p.pad_stride;
  double *basic = p.basic + (size_t)u * p.l1_stride;
  int *bl = p.blist + (size_t)u * p.pad_stride;
  for (int i = tid; i < len; i += nth) pad[i] = (i >= lag && i < lag + L) ? s4[i - lag] : 0.0;
  for (int i = tid; i < L; i += nth) basic[i] = 0.0;  // f0[i] = 0 (harvest.cpp:1176-1179)
  WB_SYNC();
  const int nsec = hv_boundaries(pad, len, bl, cnt) / 2;
  // sections are independent: thread q filters sections q, q + slots, ... in its own scratch
  const int slots = imin(p.sec_slots, nth);
  if (tid < slots) {
    double *tmp_x = p.tmp + ((size_t)u * p.sec_slots + tid) * p.seg_cap;
    for (int s = tid; s < nsec; s += slots) hv_filter_section(pad, len, bl[2 * s], bl[2 * s + 1], tmp_x, basic, lag);
  }
  WB_SYNC();
  // subsample to the requested frame period (harvest.cpp:1246-1251)
  const int nf = p.f_len[u];
  double *f0 = p.f0 + (size_t)u * p.f_stride, *ta = p.time_axis + (size_t)u * p.f_stride;
  for (int i = tid; i < nf; i += nth) {
    const double t = i * p.frame_period / 1000.0;
    ta[i] = t;
    f0[i] = basic[imin(L - 1, round_half_away(t * 1000.0))];
  }
}

// The band list of one F0 range: channel boundaries, band-pass filters (Nuttall(2 Lh + 1) * cos, GetFilteredSignal,
// harvest.cpp:99-110) and the event-list plan.  A batch with several ranges concatenates the lists of its distinct
// ranges (range groups); each list is what a call with that range alone builds.
struct HvRange {
  double f0_floor = 0.0, f0_ceil = 0.0;
  int nb = 0, max_cand = 0, max_taps = 0, nwin_max = 0;
  std::vector<double> boundary, taps;      // taps: reversed, 8 zeros after each band
  std::vector<int> tap_off, ntaps, shift;  // tap_off: into this range's taps
  std::vector<int> ecap; std::vector<long long> eoff; size_t edge_stride = 0;
};

// nullptr, or why the on-chip kernels cannot serve this range
static const char *hv_plan_range(double f0_floor, double f0_ceil, double afs, int max_ylen, bool full, HvRange *r) {
  r->f0_floor = f0_floor; r->f0_ceil = f0_ceil;
  const double adj_floor = f0_floor * 0.9, adj_ceil = f0_ceil * 1.1;
  const int nb = 1 + static_cast<int>(log(adj_ceil / adj_floor) / kLog2 * 40);
  if (nb < 3 || nb > 1024) return "Harvest: bad channel count";
  r->nb = nb;
  r->max_cand = round_half_away(nb / 10.0) * 7;
  if (r->max_cand / 7 > WB_HV_BASE) return "Harvest: f0 range too wide (more than 325 channels)";
  r->boundary.resize(nb);
  for (int i = 0; i < nb; ++i) r->boundary[i] = adj_floor * pow(2.0, (i + 1) / 40.0);
  r->tap_off.resize(nb); r->ntaps.resize(nb); r->shift.resize(nb);
  for (int i = 0; i < nb; ++i) {
    const int lh = round_half_away(afs / r->boundary[i] * 2.0);
    const int len = lh * 2 + 1;
    r->tap_off[i] = (int)r->taps.size(); r->ntaps[i] = len; r->shift[i] = lh + 1;
    std::vector<double> w(len);
    for (int j = 0; j < len; ++j) {
      const double tmp = j / (len - 1.0);
      w[j] = 0.355768 - 0.487396 * cos(2.0 * kPi * tmp) + 0.144232 * cos(4.0 * kPi * tmp) -
             0.012604 * cos(6.0 * kPi * tmp);
    }
    for (int j = -lh; j <= lh; ++j) w[j + lh] *= cos(2 * kPi * r->boundary[i] * j / afs);
    for (int j = len - 1; j >= 0; --j) r->taps.push_back(w[j]);
    for (int j = 0; j < 8; ++j) r->taps.push_back(0.0);
    if (len > r->max_taps) r->max_taps = len;
  }
  const size_t smem_sweep = sweep_smem_bytes(r->max_taps);
  const int h_max = static_cast<int>(1.5 * afs / f0_floor + 1.0);
  r->nwin_max = 2 * h_max + 1 + 2;
  int lgw = 0;
  while ((2 << lgw) <= r->nwin_max) ++lgw;
  const size_t smem_refine = (size_t)WB_HV_WARPS * 3 * r->nwin_max * 8;
  if (smem_sweep > 200 * 1024 || smem_refine > 200 * 1024 || (1 << (lgw + 2)) > WB_TW_N)
    return "Harvest: f0_floor too low for the on-chip filters";
  plan_edge_caps(r->boundary, afs, max_ylen, full, &r->ecap, &r->eoff, &r->edge_stride);
  return nullptr;
}

// Range groups of a batch: the distinct (f0_floor, f0_ceil) pairs in order of first appearance (keyed by bit pattern),
// each planned and checked against the on-chip limits when it first appears -- so an error names the first offending
// utterance.  ugrp[u] = the group of utterance u.
static int hv_make_groups(Ctx *ctx, const HarvestParams *opts, bool per_utt, int n, double afs, int max_ylen, bool full,
                          std::vector<HvRange> *groups, std::vector<int> *ugrp) {
  std::map<std::pair<unsigned long long, unsigned long long>, int> seen;
  ugrp->resize(n);
  for (int u = 0; u < n; ++u) {
    const HarvestParams &o = opts[per_utt ? u : 0];
    std::pair<unsigned long long, unsigned long long> key;
    memcpy(&key.first, &o.f0_floor, 8); memcpy(&key.second, &o.f0_ceil, 8);
    auto it = seen.find(key);
    if (it == seen.end()) {
      groups->emplace_back();
      if (const char *why = hv_plan_range(o.f0_floor, o.f0_ceil, afs, max_ylen, full, &groups->back())) {
        ctx->last_error = why;
        if (per_utt) ctx->last_error += " (utterance " + std::to_string(u) + ")";
        return 3;
      }
      it = seen.emplace(key, (int)groups->size() - 1).first;
    }
    (*ugrp)[u] = it->second;
  }
  return 0;
}

static int hv_ratio(int fs) { return imax(imin(round_half_away(fs / 8000.0), 12), 1); }   // harvest.cpp:1226, :1158

// Stage capture (test hooks, README): WB_DUMP_DECIMATED / _RAW / _BASE / _REFINED=<prefix> writes <prefix>.<chunk>
// after that stage of every chunk.  The file is "WBHVDUMP", int64 {version 1, stage 0..3, chunk, first utterance u0,
// n, ratio, nb, l1_stride, max_cand, n_groups}, double afs, int32 ugrp[n], y_len[n], l1[n], nc[n], per group
// {int32 nb, double f0_floor, double f0_ceil}, then the payload: stage 0 each utterance's y_len decimated samples,
// stage 1 raw[n][nb][l1_stride], stage 2 base[n][l1_stride][32] + int32 count[n][l1_stride], stage 3
// cand[n][l1_stride][max_cand] + score[n][l1_stride][max_cand] (before RemoveUnreliableCandidates).
// Two more capture the decision stages: WB_DUMP_CLEANED (stage 4, after harvest_remove_kernel) the cleaned cand and
// score in the stage 3 layout + base[n][l1_stride] (SearchF0Base), WB_DUMP_CONTOUR (stage 5, after
// harvest_contour_kernel) steps[n][4][l1_stride] = FixStep1 .. FixStep4 (work rows 1 .. 4; the last is what
// harvest_smooth_kernel smooths).
// WB_LOAD_REFINED=<prefix> is the way in for tests of those stages: where WB_DUMP_REFINED is written, each chunk's
// cand, score and nc are replaced by those of the stage 3 file <prefix>.<chunk>, whose n, l1_stride, max_cand and l1[]
// must be the chunk's own (anything else is an error return, never a fallback), so that harvest_remove_kernel,
// harvest_contour_kernel and harvest_smooth_kernel run, as launched here, on candidate maps the test chose.
enum { HV_DUMP_DECIMATED, HV_DUMP_RAW, HV_DUMP_BASE, HV_DUMP_REFINED, HV_DUMP_CLEANED, HV_DUMP_CONTOUR, HV_DUMP_STAGES };
struct HvDumpPart { const void *dev; size_t bytes; };

static int hv_dump(Ctx *ctx, const char *prefix, int stage, int chunk, int u0, int n, int ratio, double afs, int nb,
                   int l1_stride, int max_cand, const std::vector<int> &ugrp, const std::vector<HvRange> &groups,
                   const int *ylen_dev, const int *l1_dev, const int *nc_dev, std::vector<HvDumpPart> parts,
                   const double *y_rows = nullptr, size_t y_stride = 0) {
  std::vector<int> ylen(n), l1(n), nc(n);
  int rc = dev_sync(ctx);
  if (!rc) rc = dev_memcpy_d2h(ctx, ylen.data(), ylen_dev, (size_t)n * 4);
  if (!rc) rc = dev_memcpy_d2h(ctx, l1.data(), l1_dev, (size_t)n * 4);
  if (!rc) rc = dev_memcpy_d2h(ctx, nc.data(), nc_dev, (size_t)n * 4);
  if (!rc) rc = dev_sync(ctx);
  if (rc) return rc;
  if (y_rows)   // the decimated rows: y_rows points at utterance 0's first sample
    for (int u = 0; u < n; ++u) parts.push_back({y_rows + (size_t)u * y_stride, (size_t)ylen[u] * 8});
  std::vector<std::vector<unsigned char>> host(parts.size());
  for (size_t i = 0; i < parts.size(); ++i) {
    host[i].resize(parts[i].bytes);
    rc = dev_memcpy_d2h(ctx, host[i].data(), parts[i].dev, parts[i].bytes);
    if (rc) return rc;
  }
  rc = dev_sync(ctx);
  if (rc) return rc;
  const std::string path = std::string(prefix) + "." + std::to_string(chunk);
  FILE *f = fopen(path.c_str(), "wb");
  if (!f) { ctx->last_error = "Harvest: cannot write " + path; return 3; }
  const long long head[10] = {1, stage, chunk, u0, n, ratio, nb, l1_stride, max_cand, (long long)groups.size()};
  fwrite("WBHVDUMP", 1, 8, f);
  fwrite(head, 8, 10, f);
  fwrite(&afs, 8, 1, f);
  fwrite(ugrp.data() + u0, 4, n, f);
  fwrite(ylen.data(), 4, n, f); fwrite(l1.data(), 4, n, f); fwrite(nc.data(), 4, n, f);
  for (const HvRange &r : groups) { fwrite(&r.nb, 4, 1, f); fwrite(&r.f0_floor, 8, 1, f); fwrite(&r.f0_ceil, 8, 1, f); }
  for (const auto &h : host) fwrite(h.data(), 1, h.size(), f);
  fclose(f);
  return 0;
}

static int hv_load_refined(Ctx *ctx, const char *prefix, int chunk, int n, int l1_stride, int max_cand,
                           const int *l1_host, double *cand_dev, double *score_dev, int *nc_dev) {
  const std::string path = std::string(prefix) + "." + std::to_string(chunk);
  auto fail = [&](const char *why) { ctx->last_error = "Harvest: WB_LOAD_REFINED " + path + ": " + why; return 3; };
  FILE *f = fopen(path.c_str(), "rb");
  if (!f) return fail("cannot read");
  char magic[8];
  long long head[10];
  double afs;
  const size_t rows = (size_t)n * l1_stride * max_cand;
  std::vector<int> ints;
  std::vector<double> cs;
  const char *why = nullptr;
  if (fread(magic, 1, 8, f) != 8 || memcmp(magic, "WBHVDUMP", 8) != 0 || fread(head, 8, 10, f) != 10 ||
      fread(&afs, 8, 1, f) != 1) why = "not a WBHVDUMP file";
  else if (head[0] != 1 || head[1] != HV_DUMP_REFINED) why = "not a version 1 refined-candidates (stage 3) file";
  else if (head[4] != n || head[7] != l1_stride || head[8] != max_cand || head[9] < 0 || head[9] > 65535)
    why = "n, l1_stride or max_cand differ from the chunk's";
  if (!why) {
    ints.resize((size_t)4 * n);
    cs.resize(2 * rows);
    if (fread(ints.data(), 4, ints.size(), f) != ints.size() || fseek(f, (long)head[9] * 20, SEEK_CUR) != 0 ||
        fread(cs.data(), 8, cs.size(), f) != cs.size() || fgetc(f) != EOF) why = "payload size differs from the header's";
  }
  fclose(f);
  if (why) return fail(why);
  const int *l1 = ints.data() + 2 * (size_t)n, *nc = l1 + n;
  for (int i = 0; i < n; ++i) {
    if (l1[i] != l1_host[i]) return fail("l1[] differs from the chunk's frame counts");
    if (nc[i] < 0 || nc[i] * 7 > max_cand) return fail("nc[] out of range");
  }
  int rc = dev_memcpy_h2d(ctx, nc_dev, nc, (size_t)n * 4);
  if (!rc) rc = dev_memcpy_h2d(ctx, cand_dev, cs.data(), rows * 8);
  if (!rc) rc = dev_memcpy_h2d(ctx, score_dev, cs.data() + rows, rows * 8);
  if (!rc) rc = dev_sync(ctx);
  return rc;
}

int harvest_check_options(Ctx *ctx, int fs, const HarvestParams *opts, int n) {
  std::vector<HvRange> groups;
  std::vector<int> ugrp;
  const int ratio = hv_ratio(fs);
  return hv_make_groups(ctx, opts, true, n, static_cast<double>(fs) / ratio, 1, ratio == 1, &groups, &ugrp);
}

int harvest_run(Ctx *ctx, const Batch &b, const HarvestParams *opts, bool per_utt, double *time_axis_out,
                double *f0_out) {
  if (b.n <= 0) return 0;
  const int fs = b.fs;
  const int ratio = hv_ratio(fs);
  const double afs = static_cast<double>(fs) / ratio;
  const double frame_period = opts[0].frame_period;   // equal for every utterance (checked by the ABI layer)
  // sizes on the 1 ms grid (b.l1_host: per-utterance frame counts at 1 ms, from the ABI layer)
  const int max_ylen = static_cast<int>(ceil(static_cast<double>(b.max_x_len) / ratio));
  const int l1_stride = static_cast<int>(1000.0 * b.max_x_len / fs / 1.0) + 1;
  std::vector<HvRange> groups;
  std::vector<int> ugrp;
  const int rc0 = hv_make_groups(ctx, opts, per_utt, b.n, afs, max_ylen, ratio == 1, &groups, &ugrp);
  if (rc0) return rc0;
  // the band tables of every group one after the other; scratch strides follow the batch maxima
  const int n_groups = (int)groups.size();
  std::vector<double> taps, boundary, grp_floor(n_groups), grp_ceil(n_groups);
  std::vector<int> tap_off, ntaps, shift, ecap, grp_band0(n_groups), grp_nb(n_groups);
  std::vector<long long> eoff;
  int nb = 0, max_cand = 0, max_taps = 0, nwin_max = 0;   // batch maxima
  size_t edge_stride = 0;
  for (int g = 0; g < n_groups; ++g) {
    const HvRange &r = groups[g];
    grp_band0[g] = (int)boundary.size(); grp_nb[g] = r.nb; grp_floor[g] = r.f0_floor; grp_ceil[g] = r.f0_ceil;
    for (int i = 0; i < r.nb; ++i) tap_off.push_back((int)taps.size() + r.tap_off[i]);
    taps.insert(taps.end(), r.taps.begin(), r.taps.end());
    boundary.insert(boundary.end(), r.boundary.begin(), r.boundary.end());
    ntaps.insert(ntaps.end(), r.ntaps.begin(), r.ntaps.end());
    shift.insert(shift.end(), r.shift.begin(), r.shift.end());
    ecap.insert(ecap.end(), r.ecap.begin(), r.ecap.end());
    eoff.insert(eoff.end(), r.eoff.begin(), r.eoff.end());
    nb = imax(nb, r.nb); max_cand = imax(max_cand, r.max_cand); max_taps = imax(max_taps, r.max_taps);
    nwin_max = imax(nwin_max, r.nwin_max);
    if (r.edge_stride > edge_stride) edge_stride = r.edge_stride;
  }
  const int n_tab = (int)boundary.size();   // rows of the band tables
  const size_t smem_refine = (size_t)WB_HV_WARPS * 3 * nwin_max * 8;
  const int T = WB_SWEEP_T;
  const int padl = max_taps + 16;
  // even: with padl odd (max_taps is), every row's s(0) has the same alignment parity, so the band filters of an
  // utterance sum in the same order whatever its row and whatever else is in the batch
  const size_t y_stride = ((size_t)padl + max_ylen + 3 * T + max_taps + 64 + 1) & ~(size_t)1;
  const int lag = static_cast<int>(ceil(140.0 / ratio) * ratio);
  const size_t tmp_stride = ratio != 1 ? (size_t)b.max_x_len + 2 * lag + 32 : 0;
  const size_t pad_stride = (size_t)l1_stride + 600 + 8;
  // multi-channel storage of harvest_contour_kernel: a section takes its frames + 208.  FixStep2 keeps sections of at
  // least 7 frames (ed - st >= 6) and they lie at least one frame apart, so n sections need at most L + 208 n with
  // n <= L / 8: 27 doubles per frame.  The kernel's overflow exit is a guard, not a reachable state.
  const size_t mc_stride = (size_t)28 * l1_stride + 1024;
  const int sec_slots = 32;
  const int seg_cap = l1_stride + 600 + 8;  // a section span never exceeds the padded contour
  const size_t per_utt_bytes = y_stride * 8 + edge_stride * 8 + (size_t)nb * l1_stride * 8 +
                               (size_t)l1_stride * (WB_HV_BASE * 8 + 4) + (size_t)l1_stride * max_cand * 8 * 4 +
                               (size_t)l1_stride * (5 * 8 + 6 * 4 + 8) + mc_stride * 8 + pad_stride * (8 + 4) +
                               (size_t)sec_slots * seg_cap * 8 + tmp_stride * 16 + (size_t)nb * 20 + 1024;
  int chunk = balanced_chunk(imin(b.n, 65535), (int)dmin(65535.0, (double)ctx->scratch_budget / (double)per_utt_bytes));
#ifndef WB_EMU
  cudaFuncSetAttribute(harvest_refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_refine);
#endif
  for (int u0 = 0; u0 < b.n; u0 += chunk) {
    const int n = imin(chunk, b.n - u0);
    const char *dump[HV_DUMP_STAGES] = {getenv("WB_DUMP_DECIMATED"), getenv("WB_DUMP_RAW"), getenv("WB_DUMP_BASE"),
                                        getenv("WB_DUMP_REFINED"), getenv("WB_DUMP_CLEANED"), getenv("WB_DUMP_CONTOUR")};
    const char *load_refined = getenv("WB_LOAD_REFINED");
    ArenaPlan plan;
    const size_t o_y = plan.add((size_t)n * y_stride * 8), o_ylen = plan.add((size_t)n * 4);
    const size_t o_l1 = plan.add((size_t)n * 4), o_nc = plan.add((size_t)n * 4);
    const size_t o_nyq = plan.add((size_t)n * 32), o_nfft = plan.add((size_t)n * 4);
    const size_t o_edges = plan.add((size_t)n * edge_stride * 8);
    const size_t o_ecap = plan.add(n_tab * 4), o_eoff = plan.add(n_tab * 8);
    const size_t o_evc = plan.add((size_t)n * nb * 16), o_redo = plan.add((size_t)n * nb * 4), o_nredo = plan.add(4);
    const size_t o_raw = plan.add((size_t)n * nb * l1_stride * 8);
    const size_t o_base = plan.add((size_t)n * l1_stride * WB_HV_BASE * 8), o_bcnt = plan.add((size_t)n * l1_stride * 4);
    const size_t o_c1 = plan.add((size_t)n * l1_stride * max_cand * 8), o_s1 = plan.add((size_t)n * l1_stride * max_cand * 8);
    const size_t o_c2 = plan.add((size_t)n * l1_stride * max_cand * 8), o_s2 = plan.add((size_t)n * l1_stride * max_cand * 8);
    const size_t o_win = plan.add((size_t)hv_win_offset(nwin_max / 2 + 1) * 8);
    const size_t o_work = plan.add((size_t)n * 5 * l1_stride * 8), o_iwork = plan.add((size_t)n * 6 * l1_stride * 4);
    const size_t o_mc = plan.add((size_t)n * mc_stride * 8);
    const size_t o_pad = plan.add((size_t)n * pad_stride * 8), o_bl = plan.add((size_t)n * pad_stride * 4);
    const size_t o_stmp = plan.add((size_t)n * sec_slots * seg_cap * 8);
    const size_t o_basic = plan.add((size_t)n * l1_stride * 8);
    const size_t o_tmp = plan.add((size_t)n * tmp_stride * 8);
    const size_t o_taps = plan.add(taps.size() * 8);
    const size_t o_toff = plan.add(n_tab * 4), o_nt = plan.add(n_tab * 4), o_sh = plan.add(n_tab * 4), o_bd = plan.add(n_tab * 8);
    const size_t o_ugrp = plan.add((size_t)n * 4), o_gb0 = plan.add(n_groups * 4), o_gnb = plan.add(n_groups * 4);
    const size_t o_gfl = plan.add(n_groups * 8), o_gce = plan.add(n_groups * 8);
    const size_t o_bband = plan.add((size_t)(n + 1) * 4), o_bpair = plan.add((size_t)(n + 1) * 4);
    unsigned char *blk = arena_block(ctx, plan.total);
    if (!blk) return 2;
    double *y = (double *)(blk + o_y);
    int *ylen = (int *)(blk + o_ylen), *l1 = (int *)(blk + o_l1), *nc = (int *)(blk + o_nc);
    auto dump_stage = [&](int stage, std::vector<HvDumpPart> parts, const double *y_rows = nullptr) {
      return hv_dump(ctx, dump[stage], stage, u0 / chunk, u0, n, ratio, afs, nb, l1_stride, max_cand, ugrp, groups,
                     ylen, l1, nc, parts, y_rows, y_stride);
    };
    int rc = dev_memset(ctx, y, 0, (size_t)n * y_stride * 8);
    if (!rc) rc = dev_memset(ctx, nc, 0, (size_t)n * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, l1, b.l1_host + u0, (size_t)n * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_taps, taps.data(), taps.size() * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_toff, tap_off.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_nt, ntaps.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_sh, shift.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_bd, boundary.data(), n_tab * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_ecap, ecap.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_eoff, eoff.data(), n_tab * 8);
    // range groups of this chunk's utterances and the first block of each in the flat band / band-pair grids
    std::vector<int> bband(n + 1), bpair(n + 1);
    bband[0] = bpair[0] = 0;
    for (int i = 0; i < n; ++i) {
      const int nbu = grp_nb[ugrp[u0 + i]];
      bband[i + 1] = bband[i] + nbu;
      bpair[i + 1] = bpair[i] + (nbu + 1) / 2;
    }
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_ugrp, ugrp.data() + u0, (size_t)n * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gb0, grp_band0.data(), n_groups * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gnb, grp_nb.data(), n_groups * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gfl, grp_floor.data(), n_groups * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gce, grp_ceil.data(), n_groups * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_bband, bband.data(), (size_t)(n + 1) * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_bpair, bpair.data(), (size_t)(n + 1) * 4);
    if (rc) return rc;
    HvGroups gr;
    gr.ugrp = (const int *)(blk + o_ugrp); gr.grp_nb = (const int *)(blk + o_gnb);
    gr.grp_floor = (const double *)(blk + o_gfl); gr.grp_ceil = (const double *)(blk + o_gce);

    HvPrepParams pp;
    pp.x = b.x + (size_t)u0 * b.x_stride; pp.x_len = b.x_len + u0; pp.x_stride = b.x_stride; pp.ratio = ratio;
    pp.y = y; pp.y_stride = y_stride; pp.y_origin = padl; pp.y_len = ylen;
    if (ratio != 1) {
      DecimateParams dp;
      dp.x = pp.x; dp.x_len = pp.x_len; dp.x_stride = pp.x_stride; dp.ratio = ratio; dp.lag = lag;
      dp.tmp = (double *)(blk + o_tmp); dp.tmp_stride = tmp_stride;
      dp.y = y; dp.y_stride = y_stride; dp.y_origin = padl; dp.first = lag / ratio; dp.n_out_mode = 1;
      launch_decimate(ctx, dp, b.max_x_len, (unsigned)n);
    }
    WB_LAUNCH_COOP(harvest_prep_kernel, dim3((unsigned)n), 256, 0, ctx->stream, pp);
    if (dump[HV_DUMP_DECIMATED] && (rc = dump_stage(HV_DUMP_DECIMATED, {}, y + padl))) return rc;

    SweepParams sp;
    sp.sig = y; sp.sig_stride = y_stride; sp.sig_origin = padl; sp.y_len = ylen; sp.n_bands = nb;
    sp.taps_rev = (const double *)(blk + o_taps); sp.tap_off = (const int *)(blk + o_toff);
    sp.ntaps = (const int *)(blk + o_nt); sp.shift = (const int *)(blk + o_sh);
    sp.boundary = (const double *)(blk + o_bd); sp.afs = afs;
    sp.edges = (double *)(blk + o_edges); sp.edge_stride = edge_stride;
    sp.edge_cap = (const int *)(blk + o_ecap); sp.edge_off = (const long long *)(blk + o_eoff);
    sp.n_frames = l1; sp.frame_stride = l1_stride; sp.frame_period = 1.0;
    sp.mode = 1; sp.f0_floor = groups[0].f0_floor; sp.f0_ceil = groups[0].f0_ceil;
    if (n_groups > 1) {   // one group: bands 0 .. nb - 1 of the tables and the (band, utterance) grid, as without groups
      sp.ugrp = gr.ugrp; sp.grp_band0 = (const int *)(blk + o_gb0); sp.grp_nb = gr.grp_nb;
      sp.grp_floor = gr.grp_floor; sp.grp_ceil = gr.grp_ceil;
      sp.blk0_band = (const int *)(blk + o_bband); sp.blk0_pair = (const int *)(blk + o_bpair);
      sp.n_blk_band = bband[n]; sp.n_blk_pair = bpair[n]; sp.n_utts = n;
    }
    sp.nyq = nullptr; sp.ripple = 0;
    if (ratio == 1 && !getenv("WB_NO_RIPPLE")) {
      // Input not decimated (fs below 12 kHz): exact zeros in the waveform reach the band filters, and there the
      // ripple of the reference's mirroring loop (harvest.cpp:122-135; see nyquist_bins_kernel) is all its
      // filtered signal consists of.  1e-20 of a real signal, so the decimated rates skip it.
      std::vector<int> nfft(n);
      for (int i = 0; i < n; ++i) {
        const int xl = b.x_len_host ? b.x_len_host[u0 + i] : b.x_stride;
        const int yl = static_cast<int>(ceil(static_cast<double>(xl) / ratio));
        const int sample = yl + 5 + 2 * static_cast<int>(2.0 * afs / groups[ugrp[u0 + i]].boundary[0]);
        nfft[i] = static_cast<int>(pow(2.0, static_cast<int>(log(static_cast<double>(sample)) / kLog2) + 1.0));
      }
      rc = dev_memcpy_h2d(ctx, blk + o_nfft, nfft.data(), (size_t)n * 4);
      if (rc) return rc;
      NyquistParams np_;
      np_.sig = y; np_.stride = y_stride; np_.origin = padl; np_.y_len = ylen; np_.c = 0;
      np_.nfft = (const int *)(blk + o_nfft); np_.nyq = (double *)(blk + o_nyq);
      launch_nyquist_bins(ctx, np_, (unsigned)n);
      sp.nyq = (const double *)(blk + o_nyq); sp.ripple = 1;
    }
    sp.cand = (double *)(blk + o_raw); sp.score = nullptr;
    sp.max_taps = max_taps; sp.status = ctx->status_dev;
    sp.ev_count = (int *)(blk + o_evc); sp.redo_list = (int *)(blk + o_redo); sp.redo_count = (int *)(blk + o_nredo);
    if (!sp.ripple && !getenv("WB_SWEEP_STREAMING") && fe_smem_bytes(max_taps) <= 200 * 1024) {
      // decimated input (every rate from 12 kHz up): FIR + events, then interpolation (wb_f0common.cu)
      rc = dev_memset(ctx, sp.redo_count, 0, 4);
      if (rc) return rc;
      launch_band_sweep_split(ctx, sp, (unsigned)n);
    } else {
      launch_band_sweep(ctx, sp, (unsigned)n);
    }

    if (dump[HV_DUMP_RAW] && (rc = dump_stage(HV_DUMP_RAW, {{sp.cand, (size_t)n * nb * l1_stride * 8}}))) return rc;
    const long long slots = (long long)n * l1_stride;
    HvDetectParams dp;
    dp.raw = sp.cand; dp.n_bands = nb; dp.l1_stride = l1_stride; dp.l1 = l1; dp.gr = gr;
    dp.base = (double *)(blk + o_base); dp.base_count = (int *)(blk + o_bcnt); dp.nc = nc; dp.n_utts = n;
    WB_LAUNCH_FLAT(harvest_detect_kernel, dim3((unsigned)((slots + 127) / 128)), 128, 0, ctx->stream, dp);

    if (dump[HV_DUMP_BASE] && (rc = dump_stage(HV_DUMP_BASE, {{dp.base, (size_t)slots * WB_HV_BASE * 8},
                                                              {dp.base_count, (size_t)slots * 4}})))
      return rc;
    HvRefineParams rp;
    rp.y = y; rp.y_stride = y_stride; rp.y_origin = padl; rp.y_len = ylen; rp.afs = afs;
    rp.base = dp.base; rp.nc = nc; rp.l1_stride = l1_stride; rp.l1 = l1; rp.max_cand = max_cand;
    rp.gr = gr;
    rp.cand = (double *)(blk + o_c1); rp.score = (double *)(blk + o_s1); rp.tw = ctx->twiddle; rp.nwin_max = nwin_max;
#ifdef WB_EMU
    const unsigned refine_blocks = (unsigned)l1_stride;
#else
    const unsigned refine_blocks = (unsigned)((l1_stride + WB_HV_WARPS - 1) / WB_HV_WARPS);
#endif
    const int frame_samples = static_cast<int>(afs / 1000.0);
    if (!getenv("WB_NO_REFINE_CHAIN") && frame_samples >= 1 && frame_samples * 1000.0 == afs) {
      // slots without an in-range source frame keep these zeros
      rc = dev_memset(ctx, rp.cand, 0, (size_t)n * l1_stride * max_cand * 8);
      if (!rc) rc = dev_memset(ctx, rp.score, 0, (size_t)n * l1_stride * max_cand * 8);
      if (rc) return rc;
      HvWindowParams wp;
      wp.win = (double *)(blk + o_win); wp.afs = afs;
      WB_LAUNCH_FLAT(harvest_window_table_kernel, dim3((unsigned)(nwin_max / 2 + 1)), 128, 0, ctx->stream, wp);
      HvChainParams chp;
      chp.r = rp; chp.frame_samples = frame_samples; chp.win = wp.win;
      const size_t smem_chain = (size_t)WB_HV_WARPS * hv_chain_seg(nwin_max, frame_samples) * 8;
#ifndef WB_EMU
      cudaFuncSetAttribute(harvest_refine_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_chain);
#endif
      WB_LAUNCH_COOP(harvest_refine_chain_kernel, dim3(refine_blocks, (unsigned)n), 32 * WB_HV_WARPS, smem_chain, ctx->stream, chp);
    } else {
      WB_LAUNCH_COOP(harvest_refine_kernel, dim3(refine_blocks, (unsigned)n), 32 * WB_HV_WARPS, smem_refine, ctx->stream, rp);
    }
    if (dump[HV_DUMP_REFINED] && (rc = dump_stage(HV_DUMP_REFINED, {{rp.cand, (size_t)slots * max_cand * 8},
                                                                    {rp.score, (size_t)slots * max_cand * 8}})))
      return rc;
    if (load_refined && (rc = hv_load_refined(ctx, load_refined, u0 / chunk, n, l1_stride, max_cand, b.l1_host + u0,
                                              rp.cand, rp.score, nc)))
      return rc;

    HvRemoveParams mp;
    mp.cand_in = rp.cand; mp.score_in = rp.score; mp.cand = (double *)(blk + o_c2); mp.score = (double *)(blk + o_s2);
    mp.nc = nc; mp.l1 = l1; mp.l1_stride = l1_stride; mp.max_cand = max_cand; mp.n_utts = n;
    mp.f0_base = (double *)(blk + o_work);
#ifdef WB_EMU
    const unsigned remove_blocks = (unsigned)slots;
#else
    const unsigned remove_blocks = (unsigned)((slots + WB_RM_WARPS - 1) / WB_RM_WARPS);
#endif
    WB_LAUNCH_COOP(harvest_remove_kernel, dim3(remove_blocks), 32 * WB_RM_WARPS, 0, ctx->stream, mp);
    if (dump[HV_DUMP_CLEANED]) {
      std::vector<HvDumpPart> parts = {{mp.cand, (size_t)slots * max_cand * 8}, {mp.score, (size_t)slots * max_cand * 8}};
      for (int i = 0; i < n; ++i) parts.push_back({mp.f0_base + (size_t)i * 5 * l1_stride, (size_t)l1_stride * 8});
      if ((rc = dump_stage(HV_DUMP_CLEANED, parts))) return rc;
    }

    HvContourParams cp;
    cp.cand = mp.cand; cp.score = mp.score; cp.nc = nc; cp.l1 = l1; cp.l1_stride = l1_stride; cp.max_cand = max_cand;
    cp.work = (double *)(blk + o_work); cp.iwork = (int *)(blk + o_iwork); cp.mc = (double *)(blk + o_mc);
    cp.mc_stride = mc_stride; cp.status = ctx->status_dev;
    WB_LAUNCH_COOP(harvest_contour_kernel, dim3((unsigned)n), 128, 0, ctx->stream, cp);
    if (dump[HV_DUMP_CONTOUR]) {
      std::vector<HvDumpPart> parts;
      for (int i = 0; i < n; ++i) parts.push_back({cp.work + ((size_t)i * 5 + 1) * l1_stride, (size_t)4 * l1_stride * 8});
      if ((rc = dump_stage(HV_DUMP_CONTOUR, parts))) return rc;
    }

    HvSmoothParams hp;
    hp.work = cp.work; hp.l1_stride = l1_stride; hp.l1 = l1; hp.padded = (double *)(blk + o_pad);
    hp.tmp = (double *)(blk + o_stmp); hp.blist = (int *)(blk + o_bl); hp.basic = (double *)(blk + o_basic);
    hp.pad_stride = pad_stride; hp.sec_slots = sec_slots; hp.seg_cap = seg_cap; hp.f_len = b.f_len + u0; hp.f_stride = b.f_stride;
    hp.frame_period = frame_period;
    hp.time_axis = time_axis_out + (size_t)u0 * b.f_stride; hp.f0 = f0_out + (size_t)u0 * b.f_stride;
    WB_LAUNCH_COOP(harvest_smooth_kernel, dim3((unsigned)n), 128, 0, ctx->stream, hp);
    rc = dev_check(ctx, "harvest");
    if (rc) return rc;
  }
  return 0;
}

}  // namespace wb
