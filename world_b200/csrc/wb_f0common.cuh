// wb_f0common.cuh -- building blocks shared by the two F0 estimators (DIO and Harvest):
//   * decimate(): MATLAB-style zero-phase IIR decimator (matlabfunctions.cpp:27-125, 178-204)
//   * band sweep: one CTA per (utterance, band) runs the band's FIR over the whole utterance in
//     shared-memory tiles and picks the four zero-crossing event trains on the fly
//     (dio.cpp:296-435 / harvest.cpp:99-238), then interpolates the trains onto the frame grid
//     (interp1 of dio.cpp:471-519 / harvest.cpp:262-298).
//
// The reference filters with whole-utterance FFTs (2^17..2^21 points) - far beyond shared
// memory.  Its filters are short FIRs (<= ~1000 taps), its FFT size is chosen so that the
// circular convolution never wraps (dio.cpp:592-594, harvest.cpp:1164-1165), and the spectral
// mirroring quirk is inert for Harvest's long band-pass filters (SURVEY.md App. B5), so
// the filtered signal IS the linear convolution; it is evaluated directly: register-tiled FP64 FMA
// in the streaming sweep, FP64 tensor-core MMA (polyphase, band_fir_events_kernel) for Harvest on
// decimated input.  Filter taps are computed on the host with the same libm expressions as the
// reference and uploaded.  Where it matters the ripple the mirroring loop leaves behind IS added
// (nyquist_bins_kernel, band_sweep_ripple_kernel): DIO always -- it decides what the reference sees in digital
// silence and under heavy decimation -- and Harvest when its input is not decimated.
#pragma once
#include "wb_platform.cuh"
#include "wb_block.cuh"
#include <array>
#include <functional>
#include <vector>

namespace wb {

struct Ctx;

#define WB_SWEEP_T 2048      // outputs per tile
#define WB_SWEEP_R 8         // outputs per thread group (register tile)
#define WB_SWEEP_THREADS 256 // = T / R

// padded shared layout: one spare double per 8 keeps stride-8 accesses conflict free
WB_DEV int pad8(int i) { return i + (i >> 3); }

// ------------------------------------------------------------------------------ decimate
// IIR coefficients per ratio (matlabfunctions.cpp:29-113); unsupported ratios give zeros like
// the reference's default branch.
WB_HD inline void decimate_coefficients(int r, double a[3], double b[2]) {
  switch (r) {
    case 11: a[0] = 2.450743295230728; a[1] = -2.06794904601978; a[2] = 0.59574774438332101;
      b[0] = 0.0026822508007163792; b[1] = 0.0080467524021491377; break;
    case 12: a[0] = 2.4981398605924205; a[1] = -2.1368928194784025; a[2] = 0.62187513816221485;
      b[0] = 0.0021097275904709001; b[1] = 0.0063291827714127002; break;
    case 10: a[0] = 2.3936475118069387; a[1] = -1.9873904075111861; a[2] = 0.5658879979027055;
      b[0] = 0.0034818622251927556; b[1] = 0.010445586675578267; break;
    case 9: a[0] = 2.3236003491759578; a[1] = -1.8921545617463598; a[2] = 0.53148928133729068;
      b[0] = 0.0046331164041389372; b[1] = 0.013899349212416812; break;
    case 8: a[0] = 2.2357462340187593; a[1] = -1.7780899984041358; a[2] = 0.49152555365968692;
      b[0] = 0.0063522763407111993; b[1] = 0.019056829022133598; break;
    case 7: a[0] = 2.1225239019534703; a[1] = -1.6395144861046302; a[2] = 0.44469707800587366;
      b[0] = 0.0090366882681608418; b[1] = 0.027110064804482525; break;
    case 6: a[0] = 1.9715352749512141; a[1] = -1.4686795689225347; a[2] = 0.3893908434965701;
      b[0] = 0.013469181309343825; b[1] = 0.040407543928031475; break;
    case 5: a[0] = 1.7610939654280557; a[1] = -1.2554914843859768; a[2] = 0.3237186507788215;
      b[0] = 0.021334858522387423; b[1] = 0.06400457556716227; break;
    case 4: a[0] = 1.4499664446880227; a[1] = -0.98943497080950582; a[2] = 0.24578252340690215;
      b[0] = 0.036710750339322612; b[1] = 0.11013225101796784; break;
    case 3: a[0] = 0.95039378983237421; a[1] = -0.67429146741526791; a[2] = 0.15412211621346475;
      b[0] = 0.071221945171178636; b[1] = 0.21366583551353591; break;
    case 2: a[0] = 0.041156734567757189; a[1] = -0.42599112459189636; a[2] = 0.041037215479961225;
      b[0] = 0.16797464681802227; b[1] = 0.50392394045406674; break;
    default: a[0] = a[1] = a[2] = 0.0; b[0] = b[1] = 0.0;
  }
}

// ------------------------------------------------------------------------------ plain FIR
// out(q) = sum_k h[k] * in(q - k), q in [0, q_len[u]); `in` is zero padded on both sides.
// grid (tiles, utterances); same register tiling as the band sweep.
struct FirParams {
  const double *in; size_t in_stride; int in_origin;
  double *out; size_t out_stride; int out_origin;
  const int *base_len; int extra_len;   // q_len[u] = base_len[u] + extra_len
  const double *taps_rev; int ntaps;
};

WB_HD inline size_t fir_plain_smem_bytes(int ntaps) {
  const int seg = 2048 + ntaps + 16;
  return (size_t)(seg + (seg >> 3) + 8) * 8 + (size_t)(ntaps + 8) * 8;
}

// ------------------------------------------------------------------------------ band sweep
struct SweepParams {
  const double *sig; size_t sig_stride; int sig_origin;  // sig[u*stride + origin + m] = s(m), zero padded
  const int *y_len;                                      // [n] samples to filter per utterance
  int n_bands;
  const double *taps_rev; const int *tap_off; const int *ntaps; const int *shift;  // per band
  const double *boundary;                                // per band boundary f0
  double afs;                                            // sampling rate of sig
  double *edges; size_t edge_stride;                     // per utterance; band b: 4 trains of edge_cap[b] at edge_off[b]
  const int *edge_cap; const long long *edge_off;
  const int *n_frames; int frame_stride; double frame_period;  // frame grid: t_i = i*frame_period/1000
  int mode;                                              // 0 = DIO (candidate + score), 1 = Harvest
  const double *nyq; int ripple;                         // ripple = 1: [n][4] from nyquist_bins_kernel, band_sweep_ripple_kernel runs
  double f0_floor, f0_ceil;
  double *cand; double *score;                           // [(u*nb+b)][frame_stride]
  int max_taps;
  int *status;
  int debug_skip;   // experiments only: 1 = no candidate phase, 2 = no event phase either
  // round 2, Harvest on decimated input: the sweep is split into band_fir_events_kernel (FIR + the four event trains,
  // complete edge lists to global memory) and band_interp_kernel (edge lists -> candidates on the frame grid).
  int *ev_count;          // [n][n_bands][4] events per train; ev_count[..][0] = -1 marks a band whose lists overflowed
  int *redo_list; int *redo_count;   // (utterance * n_bands + band) pairs for the streaming kernel (history rings)
  // One F0 range per utterance (Harvest and DIO).  The per-band tables above (taps, tap_off, ntaps, shift, boundary, edge_cap,
  // edge_off) hold the band lists of every range group of the batch one after the other; utterance u uses group
  // g = ugrp[u]: bands grp_band0[g] .. grp_band0[g] + grp_nb[g] - 1 of the tables, floor / ceiling grp_floor[g] /
  // grp_ceil[g].  Band indices b elsewhere (cand rows, ev_count, redo_list) are the utterance's own 0 .. grp_nb - 1,
  // strided by n_bands = the batch maximum.  The grids are flat over the utterances' own bands (band pairs for
  // band_fir_events_kernel): blk0_band[u] / blk0_pair[u] is the first block of utterance u ([n_utts + 1] prefix sums,
  // totals n_blk_band / n_blk_pair), so the work follows the sum of the channel counts, not n x the largest.
  // ugrp == nullptr (one range for the batch): bands 0 .. n_bands - 1 and f0_floor / f0_ceil for every utterance, grid
  // (band, utterance).
  const int *ugrp = nullptr; const int *grp_band0 = nullptr, *grp_nb = nullptr;
  const double *grp_floor = nullptr, *grp_ceil = nullptr;
  const int *blk0_band = nullptr, *blk0_pair = nullptr; int n_blk_band = 0, n_blk_pair = 0, n_utts = 0;
};

// the band list of utterance u (see SweepParams::ugrp); grp = -1 without range groups.  The thresholds are read where
// they are used (sweep_store_candidate): a kernel keeps one int live, not two doubles.
struct UttBands { int band0, nb, grp; };
WB_DEV UttBands utt_bands(const SweepParams &p, int u) {
  UttBands r;
  if (!p.ugrp) { r.band0 = 0; r.nb = p.n_bands; r.grp = -1; return r; }
  r.grp = p.ugrp[u];
  r.band0 = p.grp_band0[r.grp]; r.nb = p.grp_nb[r.grp];
  return r;
}

// flat grid: the utterance u with first[u] <= blk < first[u + 1] (first[0] = 0, nondecreasing) and blk's index in it
WB_DEV int flat_block(const int *first, int n_utts, int blk, int *u) {
  int lo = 0, hi = n_utts - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= blk) lo = mid; else hi = mid - 1;
  }
  *u = lo;
  return blk - first[lo];
}

// band_fir_events_kernel: tiles of 1024 outputs = 8 outputs per event thread x 128 = 64 FIR rows of 16 outputs
// (m16n8k8 row tiles), two per filter warp.  Two input segments (TMA double buffer), the taps of two bands with 8
// leading zeros and zero padding to K + 16 (the polyphase B operand reads h[k - p] for k - p in [-8, K + 8)), two
// filtered tiles in the pad8 layout (the event threads read 8 outputs each: stride 9 doubles, conflict free; 8
// doubles ahead of each tile hold the carry), two sets of per-warp event lists.
#define WB_FE_R 8
#define WB_FE_TILE (WB_FE_R * 128)
#define WB_FE_EVMAX 16   // events of one group (8 positions, four trains) at most: 4 per train
WB_HD inline int fe_kpad(int ntaps) { return (ntaps + 8 + 7) / 8 * 8; }   // >= 8 ceil((K + 1 + 7) / 8), see fe_fir_warp
WB_HD inline int fe_seg_doubles(int max_taps) { return WB_FE_TILE + fe_kpad(max_taps) + 16; }    // even
WB_HD inline int fe_hrev_doubles(int max_taps) { return fe_kpad(max_taps) + 16; }
WB_HD inline int fe_st_doubles() { return WB_FE_TILE + (WB_FE_TILE >> 3) + 8; }
WB_HD inline size_t fe_smem_bytes(int max_taps) {
  // two segments, the taps of two bands, two filtered tiles, 2 x 4 warp counts, two mbarriers, 2 x 4 event lists of
  // 32 WB_FE_EVMAX 16-bit entries
  return (size_t)(2 * fe_seg_doubles(max_taps) + 2 * fe_hrev_doubles(max_taps) + 2 * fe_st_doubles() + 8 + 2 + 6) * 8 +
         (size_t)2 * 128 * WB_FE_EVMAX * 2;
}

WB_HD inline size_t sweep_smem_bytes(int max_taps) {
  const int seg = WB_SWEEP_T + max_taps + 16;
  return (size_t)(seg + (seg >> 3) + 8) * 8 + (size_t)(max_taps + 8) * 8 + (size_t)(WB_SWEEP_T + 8 + ((WB_SWEEP_T + 8) >> 3) + 8) * 8 +
         (size_t)(WB_SWEEP_T / WB_SWEEP_R + 40) * 8 + 8 * 256 * 8 + 2 * 256 * 8;
}

// ------------------------------------------------------------------------------ blocked decimate
// GPU restatement of decimate(): the zero-phase IIR (poles |z| <= 0.89 for every supported
// ratio) forgets its state to below 1e-19 within 384 samples, so each thread filters one block of
// DEC_BLOCK samples after a DEC_WARM sample run-in from zero state (the first block starts at
// sample 0 from zero state exactly like the reference).  Forward pass -> tmp, backward pass picks
// every r-th sample straight into the output.
#define WB_DEC_BLOCK 256
#define WB_DEC_WARM 512
struct DecimateParams {
  const double *x; const int *x_len; int x_stride;
  int ratio, lag;              // virtual edge padding of `lag` samples on both sides (Harvest), 0 for DIO
  double *tmp; size_t tmp_stride;   // forward-filtered extended signal, n + 2 lag + 18 per utterance
  double *y; size_t y_stride; int y_origin;
  int first;                   // decimated index of y[0]
  int n_out_mode;              // 0: 1 + n / r samples (DIO), 1: ceil(n / r) samples (Harvest)
};

// launchers (wb_f0common.cu)
void launch_decimate(Ctx *ctx, const DecimateParams &p, int max_x_len, unsigned n_utts);
void launch_fir_plain(Ctx *ctx, const FirParams &p, unsigned tiles, unsigned n_utts);
void launch_band_sweep(Ctx *ctx, const SweepParams &p, unsigned n_utts);
// Harvest, decimated input: FIR + events, interpolation, then the streaming kernel for the bands whose lists overflowed
void launch_band_sweep_split(Ctx *ctx, const SweepParams &p, unsigned n_utts);

// the two spectrum bins the reference's mirroring loop corrupts (see nyquist_bins_kernel)
struct NyquistParams {
  const double *sig; size_t stride; int origin;      // sig[u*stride + origin + q], time index n = q - c
  const int *y_len; int c;                           // q in [0, y_len[u] + 2 c)
  const int *nfft;                                   // [n] reference FFT size per utterance
  double *nyq;                                       // out [n][4]: Re Ys[N/2-1], Im Ys[N/2-1], Ys[N/2], N
};
void launch_nyquist_bins(Ctx *ctx, const NyquistParams &p, unsigned n_utts);

// ------------------------------------------------------------------------------ band plan (host)
// One F0 range per utterance (Harvest and DIO): the batch's distinct ranges are range groups, in order of first
// appearance.  Their band lists are concatenated into one set of tables, and each utterance reaches its bands through
// its group index (SweepParams::ugrp).  Each list is what a call with that range alone builds.
struct BandList {
  double f0_floor = 0.0, f0_ceil = 0.0;
  int nb = 0, max_taps = 0;
  std::vector<double> boundary, taps;      // taps: reversed, 8 zeros after each band
  std::vector<int> tap_off, ntaps, shift;  // tap_off: into this list's taps
};
struct RangeGroups {
  std::vector<BandList> lists;   // one per group
  std::vector<int> ugrp;         // [n] the group of each utterance
};
// Groups n utterances by key(i), the doubles that fix option i's band list, compared by bit pattern (per_utt: option u
// is utterance u's, else option 0 serves every utterance).  build(i, list) makes the list when its key first appears and
// returns nullptr, or why the on-chip kernels cannot serve it: then 3 (EINVAL) with that reason in last_error and, per
// utterance, " (utterance u)" after it.  So an error names the first bad utterance.
int group_ranges(Ctx *ctx, int n, bool per_utt, const std::function<std::array<double, 3>(int)> &key,
                 const std::function<const char *(int, BandList *)> &build, RangeGroups *g);

// a chunk's device copy of the group tables (BandTables::upload), set with one group too
struct GroupTables { const int *ugrp, *grp_nb; const double *grp_floor, *grp_ceil; };

// The band tables of a batch: every group's list one after the other, with its event lists planned for the batch's
// longest decimated utterance (max_ylen; full: keep every event), and the group tables.  Scratch strides follow the
// batch maxima.
struct BandTables {
  BandTables(const RangeGroups &g, double afs, int max_ylen, bool full);
  std::vector<int> ugrp;
  std::vector<double> taps, boundary, grp_floor, grp_ceil;
  std::vector<int> tap_off, ntaps, shift, ecap, grp_band0, grp_nb;
  std::vector<long long> eoff;
  int nb = 0, max_taps = 0;   // batch maxima
  size_t edge_stride = 0;
  // A chunk of n utterances: the bytes of its copy in the chunk's block, then the copy itself at blk, enqueued on
  // ctx->stream: the tables, and utterances [u0, u0 + n)'s group indices and the prefix sums of their bands and band
  // pairs.  upload fills sp's table and group fields.  With one group sp.ugrp stays null and the sweep runs on the
  // (band, utterance) grid.
  size_t chunk_bytes(int n) const;
  int upload(Ctx *ctx, unsigned char *blk, int u0, int n, SweepParams *sp, GroupTables *gt = nullptr) const;
 private:
  struct Part { const void *src; size_t bytes; };
  std::vector<Part> chunk_parts(int u0, int n, const int *bband, const int *bpair) const;
};

}  // namespace wb
