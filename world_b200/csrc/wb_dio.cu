// wb_dio.cu -- DIO F0 estimation for a batch (replaces Dio()/DioGeneralBody, dio.cpp:578-648).
// Algorithm card: SURVEY.md A3.
//   K-DIOp  dio_prep_kernel      decimate (optional) + DC removal                (dio.cpp:60-79)
//   fir_plain_kernel             zero-phase 50 Hz low-cut FIR                     (dio.cpp:40-53, 86-104)
//   K-DIOf  band_sweep_kernel    per band Nuttall low-pass + 4 zero-crossing trains + interp1 onto
//                                the frame grid -> candidates and scores           (dio.cpp:296-568)
//   K-DIOc  dio_contour_kernel   best candidate + FixStep1..4                     (dio.cpp:112-289)
// Host side computes every size and filter tap with the reference's own double-precision
// expressions (and the host libm), so frame counts, band lists and taps are bit-identical.
// One option per utterance (world_b200_dio_batch_options): the batch's distinct band lists are range groups whose
// tables are concatenated; the sweep runs on a flat grid over the utterances' own bands and the contour takes each
// utterance's band count, floor and allowed_range.  speed and frame_period are shared by the batch.
#include "wb_internal.h"
#include "wb_f0common.cuh"
#include <stdlib.h>
#include <string.h>
#include <array>
#include <map>
#include <string>
#include <vector>

namespace wb {

// Event-list capacity per band and train: crossings of a signal band-limited around/below
// `boundary` cannot be denser than ~boundary per second for long; 2.5x margin, hard bound
// ylen/2+2 (a negative-going crossing needs two samples).  The lists are history rings: more events
// than this wrap around; only a look-back beyond the last `cap` events raises status bit 4.
static void plan_edge_caps(const std::vector<double> &boundary, double afs, int max_ylen,
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
    // DIO keeps every event: with the mirroring ripple in, digital silence makes the difference trains fire
    // every sample while the crossing trains may stay silent, so frames cannot be finalised until the silence
    // ends and the look-back is as long as the silence (few bands, so the full lists are affordable)
    soft = hard;
    (*cap)[i] = (int)(soft < hard ? soft : hard);
    (*off)[i] = run;
    run += 4LL * (*cap)[i];
  }
  *stride = (size_t)run;
}

struct DioPrepParams {
  const double *x; const int *x_len; int x_stride;
  int ratio;
  double *y; size_t y_stride; int y_origin;   // mean-removed signal, zero padded
  int *y_len;                                  // out: 1 + x_len / ratio
};

WB_KERNEL(256, 2) dio_prep_kernel(DioPrepParams p) {
  WB_SHARED double red[WB_RED_DOUBLES];
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int n = p.x_len[u];
  const double *x = p.x + (size_t)u * p.x_stride;
  double *y = p.y + (size_t)u * p.y_stride + p.y_origin;
  const int ylen = 1 + n / p.ratio;
  if (p.ratio != 1) {
    // launch_decimate() already left (n-1)/r+1 (+ a few mirrored-edge) samples in y; the rest of y
    // stays zero (dio.cpp:67-73)
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

struct DioContourParams {
  const double *cand; const double *score; int n_bands; int frame_stride;   // rows [n][n_bands = batch maximum][stride]
  const int *f_len; double frame_period, f0_floor, allowed_range;
  // one option per utterance: range group ugrp[u] (its band count and floor; nullptr: n_bands and f0_floor for every
  // utterance) and allowed[u] (nullptr: allowed_range for every utterance)
  const int *ugrp; const int *grp_nb; const double *grp_floor; const double *allowed;
  double *work;      // [n][4][frame_stride]
  int *sections;     // [n][2][frame_stride]
  double *time_axis; double *f0; int out_stride;
};

WB_DEV double dio_select_best(double cur, double past, const double *cand, int nb, int stride, int target,
                              double allowed) {
  const double reference = (cur * 3.0 - past) / 2.0;
  double best = cand[target];
  double min_err = fabs(reference - best);
  for (int b = 1; b < nb; ++b) {
    const double c = cand[(size_t)b * stride + target];
    const double e = fabs(reference - c);
    if (e < min_err) { min_err = e; best = c; }
  }
  if (fabs(1.0 - best / reference) > allowed) return 0.0;
  return best;
}

WB_KERNEL(256, 2) dio_contour_kernel(DioContourParams p) {
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int L = p.f_len[u], fstr = p.frame_stride;
  const int nb = p.ugrp ? p.grp_nb[p.ugrp[u]] : p.n_bands;
  const double f0_floor = p.ugrp ? p.grp_floor[p.ugrp[u]] : p.f0_floor;
  const double allowed_range = p.allowed ? p.allowed[u] : p.allowed_range;
  const double *cand = p.cand + (size_t)u * p.n_bands * fstr;
  const double *score = p.score + (size_t)u * p.n_bands * fstr;
  double *best = p.work + (size_t)u * 4 * fstr, *s1 = best + fstr, *s2 = s1 + fstr, *s3 = s2 + fstr;
  int *pos = p.sections + (size_t)u * 2 * fstr, *neg = pos + fstr;
  double *f0 = p.f0 + (size_t)u * p.out_stride, *ta = p.time_axis + (size_t)u * p.out_stride;
  for (int i = tid; i < L; i += nth) {
    ta[i] = i * p.frame_period / 1000.0;  // dio.cpp:609-610
    double bs = score[i], bf = cand[i];
    for (int b = 1; b < nb; ++b) {
      const double sc = score[(size_t)b * fstr + i];
      if (bs > sc) { bs = sc; bf = cand[(size_t)b * fstr + i]; }
    }
    best[i] = bf;
    f0[i] = 0.0;
  }
  const int vrm = static_cast<int>(0.5 + 1000.0 / p.frame_period / f0_floor) * 2 + 1;
  if (L <= vrm) return;  // dio.cpp:266 (the reference leaves f0 unwritten; zeros here)
  WB_SYNC();
  // step 1: s1 (f0_base is `best` with the first/last vrm frames zeroed)
  for (int i = tid; i < L; i += nth) {
    double v = 0.0;
    if (i >= vrm) {
      const double bi = (i < L - vrm) ? best[i] : 0.0;
      const double bp = (i - 1 >= vrm && i - 1 < L - vrm) ? best[i - 1] : 0.0;
      v = fabs((bi - bp) / (kTiny + bi)) < allowed_range ? bi : 0.0;
    }
    s1[i] = v;
  }
  WB_SYNC();
  const int center = (vrm - 1) / 2;
  for (int i = tid; i < L; i += nth) {
    double v = s1[i];
    if (i >= center && i < L - center)
      for (int j = -center; j <= center; ++j)
        if (s1[i + j] == 0) { v = 0.0; break; }
    s2[i] = v;
    s3[i] = v;
  }
  WB_SYNC();
  if (tid == 0) {
    int pc = 0, nc = 0;
    for (int i = 1; i < L; ++i) {
      if (s2[i] == 0 && s2[i - 1] != 0) neg[nc++] = i - 1;
      else if (s2[i - 1] == 0 && s2[i] != 0) pos[pc++] = i;
    }
    // step 3: forward extension (dio.cpp:215-231), in s3
    for (int i = 0; i < nc; ++i) {
      const int limit = i == nc - 1 ? L - 1 : neg[i + 1];
      for (int j = neg[i]; j < limit; ++j) {
        s3[j + 1] = dio_select_best(s3[j], s3[j - 1], cand, nb, fstr, j + 1, allowed_range);
        if (s3[j + 1] == 0) break;
      }
    }
    // step 4: backward extension (dio.cpp:237-253), in place on s3 (copy semantics are identical:
    // the reference copies step3 into step4 first and then only reads step4)
    for (int i = pc - 1; i >= 0; --i) {
      const int limit = i == 0 ? 1 : pos[i - 1];
      for (int j = pos[i]; j > limit; --j) {
        s3[j - 1] = dio_select_best(s3[j], s3[j + 1], cand, nb, fstr, j - 1, allowed_range);
        if (s3[j - 1] == 0) break;
      }
    }
  }
  WB_SYNC();
  for (int i = tid; i < L; i += nth) f0[i] = s3[i];
}

// The band list of one F0 range (f0_floor, f0_ceil, channels_in_octave): channel boundaries (dio.cpp:582-588), per
// band Nuttall low-pass of 4 ha taps (GetFilteredSignal, dio.cpp:296-337) and the event-list plan.  A batch with several
// ranges concatenates the lists of its distinct ranges (range groups); each list is what a call with that range alone
// builds.
struct DioRange {
  double f0_floor = 0.0, f0_ceil = 0.0;
  int nb = 0, max_taps = 0;
  std::vector<double> boundary, taps;      // taps: reversed, 8 zeros after each band
  std::vector<int> tap_off, ntaps, shift;  // tap_off: into this range's taps
  std::vector<int> ecap; std::vector<long long> eoff; size_t edge_stride = 0;
};

// nullptr, or why the on-chip kernels cannot serve this range
static const char *dio_plan_range(const DioParams &o, double afs, int max_ylen, DioRange *r) {
  r->f0_floor = o.f0_floor; r->f0_ceil = o.f0_ceil;
  const int nb = 1 + static_cast<int>(log(o.f0_ceil / o.f0_floor) / kLog2 * o.channels_in_octave);
  if (nb < 1 || nb > 4096) return "Dio: bad band count";
  r->nb = nb;
  r->boundary.resize(nb);
  for (int i = 0; i < nb; ++i) r->boundary[i] = o.f0_floor * pow(2.0, (i + 1) / o.channels_in_octave);
  r->tap_off.resize(nb); r->ntaps.resize(nb); r->shift.resize(nb);
  for (int i = 0; i < nb; ++i) {
    const int ha = round_half_away(afs / r->boundary[i] / 2.0);
    if (ha < 1) {
      // band above afs / 2 (heavy decimation): the reference's window has zero length, its filtered signal
      // is identically zero, so the band yields no events -- the same through an all-zero filter
      r->tap_off[i] = (int)r->taps.size(); r->ntaps[i] = 8; r->shift[i] = 0;
      for (int j = 0; j < 16; ++j) r->taps.push_back(0.0);
      if (8 > r->max_taps) r->max_taps = 8;
      continue;
    }
    const int len = ha * 4;
    r->tap_off[i] = (int)r->taps.size(); r->ntaps[i] = len; r->shift[i] = ha * 2;
    std::vector<double> w(len);
    for (int j = 0; j < len; ++j) {
      const double tmp = j / (len - 1.0);
      w[j] = 0.355768 - 0.487396 * cos(2.0 * kPi * tmp) + 0.144232 * cos(4.0 * kPi * tmp) -
             0.012604 * cos(6.0 * kPi * tmp);
    }
    for (int j = len - 1; j >= 0; --j) r->taps.push_back(w[j]);
    for (int j = 0; j < 8; ++j) r->taps.push_back(0.0);
    if (len > r->max_taps) r->max_taps = len;
  }
  if (sweep_smem_bytes(r->max_taps) > 200 * 1024)
    return "Dio: filters too long for shared memory (lower fs / raise f0_floor / use speed > 1)";
  plan_edge_caps(r->boundary, afs, max_ylen, &r->ecap, &r->eoff, &r->edge_stride);
  return nullptr;
}

// Range groups of a batch: the distinct (f0_floor, f0_ceil, channels_in_octave) triples in order of first appearance
// (keyed by bit pattern), each planned and checked against the on-chip limits when it first appears -- so an error
// names the first offending utterance.  ugrp[u] = the group of utterance u.  allowed_range is not part of the key: only
// the contour uses it, per utterance.
static int dio_make_groups(Ctx *ctx, const DioParams *opts, bool per_utt, int n, double afs, int max_ylen,
                           std::vector<DioRange> *groups, std::vector<int> *ugrp) {
  std::map<std::array<unsigned long long, 3>, int> seen;
  ugrp->resize(n);
  for (int u = 0; u < n; ++u) {
    const DioParams &o = opts[per_utt ? u : 0];
    std::array<unsigned long long, 3> key;
    memcpy(&key[0], &o.f0_floor, 8); memcpy(&key[1], &o.f0_ceil, 8); memcpy(&key[2], &o.channels_in_octave, 8);
    auto it = seen.find(key);
    if (it == seen.end()) {
      groups->emplace_back();
      if (const char *why = dio_plan_range(o, afs, max_ylen, &groups->back())) {
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

static int dio_ratio(int speed) { return imax(imin(speed, 12), 1); }

int dio_check_options(Ctx *ctx, int fs, const DioParams *opts, int n) {
  std::vector<DioRange> groups;
  std::vector<int> ugrp;
  return dio_make_groups(ctx, opts, true, n, static_cast<double>(fs) / dio_ratio(opts[0].speed), 1, &groups, &ugrp);
}

int dio_run(Ctx *ctx, const Batch &b, const DioParams *opts, bool per_utt, double *time_axis_out, double *f0_out) {
  if (b.n <= 0) return 0;
  const int fs = b.fs;
  // speed and frame_period: equal for every utterance (checked by the ABI layer)
  const double frame_period = opts[0].frame_period;
  const int ratio = dio_ratio(opts[0].speed);
  const double afs = static_cast<double>(fs) / ratio;
  const int max_ylen = 1 + b.max_x_len / ratio;
  std::vector<DioRange> groups;
  std::vector<int> ugrp;
  const int rc0 = dio_make_groups(ctx, opts, per_utt, b.n, afs, max_ylen, &groups, &ugrp);
  if (rc0) return rc0;
  // the band tables of every group one after the other; scratch strides follow the batch maxima
  const int n_groups = (int)groups.size();
  std::vector<double> taps, boundary, grp_floor(n_groups), grp_ceil(n_groups);
  std::vector<int> tap_off, ntaps, shift, ecap, grp_band0(n_groups), grp_nb(n_groups);
  std::vector<long long> eoff;
  int nb = 0, max_taps = 0;   // batch maxima
  size_t edge_stride = 0;
  for (int g = 0; g < n_groups; ++g) {
    const DioRange &r = groups[g];
    grp_band0[g] = (int)boundary.size(); grp_nb[g] = r.nb; grp_floor[g] = r.f0_floor; grp_ceil[g] = r.f0_ceil;
    for (int i = 0; i < r.nb; ++i) tap_off.push_back((int)taps.size() + r.tap_off[i]);
    taps.insert(taps.end(), r.taps.begin(), r.taps.end());
    boundary.insert(boundary.end(), r.boundary.begin(), r.boundary.end());
    ntaps.insert(ntaps.end(), r.ntaps.begin(), r.ntaps.end());
    shift.insert(shift.end(), r.shift.begin(), r.shift.end());
    ecap.insert(ecap.end(), r.ecap.begin(), r.ecap.end());
    eoff.insert(eoff.end(), r.eoff.begin(), r.eoff.end());
    nb = imax(nb, r.nb); max_taps = imax(max_taps, r.max_taps);
    if (r.edge_stride > edge_stride) edge_stride = r.edge_stride;
  }
  const int n_tab = (int)boundary.size();   // rows of the band tables
  // allowed_range per utterance only where it differs (it is not part of the group key)
  bool mixed_allowed = false;
  for (int u = 1; per_utt && u < b.n; ++u) mixed_allowed = mixed_allowed || !(opts[u].allowed_range == opts[0].allowed_range);
  // low-cut filter (DesignLowCutFilter, dio.cpp:40-53) as a centred FIR of 2c+1 taps
  const int c = round_half_away(afs / 50.0);
  const int nlc = 2 * c + 1;
  std::vector<double> lc(nlc);
  {
    for (int i = 1; i <= nlc; ++i) lc[i - 1] = 0.5 - 0.5 * cos(i * 2.0 * kPi / (nlc + 1));
    double sum = 0.0;
    for (int i = 0; i < nlc; ++i) sum += lc[i];
    for (int i = 0; i < nlc; ++i) lc[i] = -lc[i] / sum;
    lc[c] += 1.0;  // "low_cut_filter[0] += 1.0" after the circular shift that centres the filter
  }
  std::vector<double> lc_rev(lc.rbegin(), lc.rend());
  if (fir_plain_smem_bytes(nlc) > 200 * 1024) {
    ctx->last_error = "Dio: filters too long for shared memory (lower fs / raise f0_floor / use speed > 1)";
    return 3;
  }
  const int T = WB_SWEEP_T;
  // Every filter of the chain (decimation, low-cut FIR, band sweep, Nyquist bins) sums in an order that depends on its
  // own taps and the utterance's samples only, not on a row's alignment, so padl may follow the batch's longest filter.
  const int padl = imax(max_taps, nlc) + 16;
  const size_t y_stride = (size_t)padl + max_ylen + 2 * c + 3 * T + max_taps + nlc + 64;
  const int fstr = b.f_stride;
  const size_t tmp_stride = ratio != 1 ? (size_t)b.max_x_len + 32 : 0;
  const size_t per_utt_bytes = y_stride * 16 + edge_stride * 8 + (size_t)nb * fstr * 16 +
                               (size_t)fstr * (4 * 8 + 2 * 4) + tmp_stride * 16 + 256;
  int chunk = balanced_chunk(imin(b.n, 65535), (int)dmin(65535.0, (double)ctx->scratch_budget / (double)per_utt_bytes));
  for (int u0 = 0; u0 < b.n; u0 += chunk) {
    const int n = imin(chunk, b.n - u0);
    ArenaPlan plan;
    const size_t o_y = plan.add((size_t)n * y_stride * 8), o_ylc = plan.add((size_t)n * y_stride * 8);
    const size_t o_ylen = plan.add((size_t)n * 4), o_nyq = plan.add((size_t)n * 32), o_nfft = plan.add((size_t)n * 4);
    const size_t o_edges = plan.add((size_t)n * edge_stride * 8);
    const size_t o_ecap = plan.add(n_tab * 4), o_eoff = plan.add(n_tab * 8);
    const size_t o_cand = plan.add((size_t)n * nb * fstr * 8), o_score = plan.add((size_t)n * nb * fstr * 8);
    const size_t o_work = plan.add((size_t)n * 4 * fstr * 8), o_sec = plan.add((size_t)n * 2 * fstr * 4);
    const size_t o_tmp = plan.add((size_t)n * tmp_stride * 8);
    const size_t o_lc = plan.add(lc_rev.size() * 8 + 64), o_taps = plan.add(taps.size() * 8);
    const size_t o_toff = plan.add(n_tab * 4), o_nt = plan.add(n_tab * 4), o_sh = plan.add(n_tab * 4), o_bd = plan.add(n_tab * 8);
    const size_t o_ugrp = plan.add((size_t)n * 4), o_gb0 = plan.add(n_groups * 4), o_gnb = plan.add(n_groups * 4);
    const size_t o_gfl = plan.add(n_groups * 8), o_gce = plan.add(n_groups * 8);
    const size_t o_bband = plan.add((size_t)(n + 1) * 4), o_allow = plan.add((size_t)n * 8);
    unsigned char *blk = arena_block(ctx, plan.total);
    if (!blk) return 2;
    double *y = (double *)(blk + o_y), *ylc = (double *)(blk + o_ylc);
    int *ylen = (int *)(blk + o_ylen);
    int rc = dev_memset(ctx, y, 0, (size_t)n * y_stride * 8);
    if (!rc) rc = dev_memset(ctx, ylc, 0, (size_t)n * y_stride * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_lc, lc_rev.data(), lc_rev.size() * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_taps, taps.data(), taps.size() * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_toff, tap_off.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_nt, ntaps.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_sh, shift.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_bd, boundary.data(), n_tab * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_ecap, ecap.data(), n_tab * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_eoff, eoff.data(), n_tab * 8);
    // range groups of this chunk's utterances and the first block of each in the flat band grid
    std::vector<int> bband(n + 1, 0);
    std::vector<double> allow;
    if (n_groups > 1) {
      for (int i = 0; i < n; ++i) bband[i + 1] = bband[i] + grp_nb[ugrp[u0 + i]];
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_ugrp, ugrp.data() + u0, (size_t)n * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gb0, grp_band0.data(), n_groups * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gnb, grp_nb.data(), n_groups * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gfl, grp_floor.data(), n_groups * 8);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_gce, grp_ceil.data(), n_groups * 8);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_bband, bband.data(), (size_t)(n + 1) * 4);
    }
    if (mixed_allowed) {
      allow.resize(n);
      for (int i = 0; i < n; ++i) allow[i] = opts[u0 + i].allowed_range;
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_allow, allow.data(), (size_t)n * 8);
    }
    if (rc) return rc;

    DioPrepParams pp;
    pp.x = b.x + (size_t)u0 * b.x_stride; pp.x_len = b.x_len + u0; pp.x_stride = b.x_stride; pp.ratio = ratio;
    pp.y = y; pp.y_stride = y_stride; pp.y_origin = padl; pp.y_len = ylen;
    if (ratio != 1) {
      DecimateParams dp;
      dp.x = pp.x; dp.x_len = pp.x_len; dp.x_stride = pp.x_stride; dp.ratio = ratio; dp.lag = 0;
      dp.tmp = (double *)(blk + o_tmp); dp.tmp_stride = tmp_stride;
      dp.y = y; dp.y_stride = y_stride; dp.y_origin = padl; dp.first = 0; dp.n_out_mode = 0;
      launch_decimate(ctx, dp, b.max_x_len, (unsigned)n);
    }
    WB_LAUNCH_COOP(dio_prep_kernel, dim3((unsigned)n), 256, 0, ctx->stream, pp);

    // ylc(q) = sum_k lc[k] y(q - k), q in [0, ylen + 2c): time index n = q - c
    FirParams fp;
    fp.in = y; fp.in_stride = y_stride; fp.in_origin = padl;
    fp.out = ylc; fp.out_stride = y_stride; fp.out_origin = padl;
    fp.base_len = ylen; fp.extra_len = 2 * c; fp.taps_rev = (const double *)(blk + o_lc); fp.ntaps = nlc;
    const unsigned tiles = (unsigned)((max_ylen + 2 * c + 2047) / 2048);
    launch_fir_plain(ctx, fp, tiles, (unsigned)n);

    // the reference's FFT size per utterance: GetSuitableFFTSize(y_length + 2 c + 1 + 4 int(1 + afs / b0 / 2))
    // (dio.cpp:590-592, common.cpp:51-54), host libm like there; b0 is the first boundary of the utterance's group
    std::vector<int> nfft(n);
    for (int i = 0; i < n; ++i) {
      const int xl = b.x_len_host ? b.x_len_host[u0 + i] : b.x_stride;
      const int yl = 1 + xl / ratio;
      const double b0 = groups[ugrp[u0 + i]].boundary[0];
      const int sample = yl + c * 2 + 1 + 4 * static_cast<int>(1.0 + afs / b0 / 2.0);
      nfft[i] = static_cast<int>(pow(2.0, static_cast<int>(log(static_cast<double>(sample)) / kLog2) + 1.0));
    }
    rc = dev_memcpy_h2d(ctx, blk + o_nfft, nfft.data(), (size_t)n * 4);
    if (rc) return rc;
    NyquistParams np_;
    np_.sig = ylc; np_.stride = y_stride; np_.origin = padl; np_.y_len = ylen; np_.c = c;
    np_.nfft = (const int *)(blk + o_nfft); np_.nyq = (double *)(blk + o_nyq);
    launch_nyquist_bins(ctx, np_, (unsigned)n);

    SweepParams sp;
    sp.sig = ylc; sp.sig_stride = y_stride; sp.sig_origin = padl + c; sp.y_len = ylen; sp.n_bands = nb;
    sp.taps_rev = (const double *)(blk + o_taps); sp.tap_off = (const int *)(blk + o_toff);
    sp.ntaps = (const int *)(blk + o_nt); sp.shift = (const int *)(blk + o_sh);
    sp.boundary = (const double *)(blk + o_bd); sp.afs = afs;
    sp.edges = (double *)(blk + o_edges); sp.edge_stride = edge_stride;
    sp.edge_cap = (const int *)(blk + o_ecap); sp.edge_off = (const long long *)(blk + o_eoff);
    sp.n_frames = b.f_len + u0; sp.frame_stride = fstr; sp.frame_period = frame_period;
    sp.mode = 0; sp.f0_floor = groups[0].f0_floor; sp.f0_ceil = groups[0].f0_ceil;
    if (n_groups > 1) {   // one group: bands 0 .. nb - 1 of the tables and the (band, utterance) grid, as without groups
      sp.ugrp = (const int *)(blk + o_ugrp); sp.grp_band0 = (const int *)(blk + o_gb0); sp.grp_nb = (const int *)(blk + o_gnb);
      sp.grp_floor = (const double *)(blk + o_gfl); sp.grp_ceil = (const double *)(blk + o_gce);
      sp.blk0_band = (const int *)(blk + o_bband); sp.n_blk_band = bband[n]; sp.n_utts = n;
    }
    sp.nyq = (const double *)(blk + o_nyq); sp.ripple = getenv("WB_NO_RIPPLE") ? 0 : 1;   // A/B switch for experiments
    sp.cand = (double *)(blk + o_cand); sp.score = (double *)(blk + o_score);
    sp.max_taps = max_taps; sp.status = ctx->status_dev;
    launch_band_sweep(ctx, sp, (unsigned)n);

    DioContourParams cp;
    cp.cand = sp.cand; cp.score = sp.score; cp.n_bands = nb; cp.frame_stride = fstr; cp.f_len = b.f_len + u0;
    cp.frame_period = frame_period; cp.f0_floor = groups[0].f0_floor; cp.allowed_range = opts[0].allowed_range;
    cp.ugrp = sp.ugrp; cp.grp_nb = sp.grp_nb; cp.grp_floor = sp.grp_floor;
    cp.allowed = mixed_allowed ? (const double *)(blk + o_allow) : nullptr;
    cp.work = (double *)(blk + o_work); cp.sections = (int *)(blk + o_sec);
    cp.time_axis = time_axis_out + (size_t)u0 * b.f_stride; cp.f0 = f0_out + (size_t)u0 * b.f_stride;
    cp.out_stride = b.f_stride;
    WB_LAUNCH_COOP(dio_contour_kernel, dim3((unsigned)n), 256, 0, ctx->stream, cp);
    rc = dev_check(ctx, "dio");
    if (rc) return rc;
  }
  return 0;
}

}  // namespace wb
