// wb_chain.h -- the context behind the C ABI's handle, and the analysis chain that the device drivers (wb_api.cu) and the
// host pipelines (wb_host.cu) share: one checked plan per call, one stage sequence per slice or chunk.
#pragma once
#include "wb_internal.h"
#include "../../include/world_b200.h"

struct WorldB200 {
  wb::Ctx c;
  int *lens_dev = nullptr;
  size_t lens_cap = 0;
  // world_b200_analyze_batch: two sibling contexts ("lanes"), each with its own stream, scratch arena and staging
  // ring, created on first use; fork / join events order them against this context's stream
  WorldB200 *lane[2] = {nullptr, nullptr};
  void *lane_stream[2] = {nullptr, nullptr};   // cudaStream_t
  void *ev_fork = nullptr, *ev_join[2] = {nullptr, nullptr};   // cudaEvent_t
  // multi-GPU (wb_multi.cu): NCCL communicator + one event per utterance slice of analyze_batch_allgather
  wb::Comm *comm = nullptr;
  std::vector<void *> ev_slice;
};

namespace wb {

// What an analysis entry point receives.  x: n rows of x_stride samples, doubles (nbit 0) or little-endian PCM.  The
// per-utterance option arrays may be NULL (the AnalysisOption's own option for every utterance); at most one of the two
// F0 arrays, and the spectral arrays only with coded rows.  coded: spectrogram / aperiodicity receive dims /
// GetNumberOfAperiodicities(fs) coded values per frame instead of fft_size / 2 + 1 bins.  A NULL spectrogram or
// aperiodicity skips its stage.  f0_stride 0: rows as long as the longest utterance's frame count.  row_stride: doubles
// per frame of full rows, at least every utterance's fft_size / 2 + 1; 0 for fft_size / 2 + 1 with one option, or the
// largest size's with per-utterance options.  transform: a voice transformation, which has no analysis outputs and
// plans both spectral stages.
struct ChainRequest {
  ChainRequest(const void *x, int nbit, int n, int x_stride, const int *x_lengths, int fs,
               const WorldB200AnalysisOption *opt, double *time_axis, double *f0, int f0_stride, double *spectrogram,
               double *aperiodicity)
      : x(x), nbit(nbit), n(n), x_stride(x_stride), x_lengths(x_lengths), fs(fs), opt(opt), time_axis(time_axis),
        f0(f0), f0_stride(f0_stride), spectrogram(spectrogram), aperiodicity(aperiodicity) {}
  const void *x;
  int nbit, n, x_stride;
  const int *x_lengths;
  int fs;
  const WorldB200AnalysisOption *opt;
  double *time_axis, *f0;
  int f0_stride;
  double *spectrogram, *aperiodicity;
  bool coded = false;
  int dims = 0;
  const HarvestOption *harvest_options = nullptr;
  const DioOption *dio_options = nullptr;
  const CheapTrickOption *cheaptrick_options = nullptr;
  const D4COption *d4c_options = nullptr;
  int row_stride = 0;
  // packed layout (the *_packed entry points): utterance u is samples [x_offsets[u], x_offsets[u + 1]) of x (HOST,
  // n + 1 offsets); x_stride, x_lengths and f0_stride are unused, and the outputs are [F] frames, utterance u's from
  // the plan's f_off[u]
  bool packed = false;
  const long long *x_offsets = nullptr;
  bool transform = false;
};

// The request of a coded-row entry point: number_of_dimensions coded values per spectral frame.
inline ChainRequest coded_request(const void *x, int nbit, int n, int x_stride, const int *x_lengths, int fs,
                                  const WorldB200AnalysisOption *opt, int number_of_dimensions, double *time_axis,
                                  double *f0, int f0_stride, double *coded_spectral_envelope,
                                  double *coded_aperiodicity) {
  ChainRequest r(x, nbit, n, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, coded_spectral_envelope,
                 coded_aperiodicity);
  r.coded = true;
  r.dims = number_of_dimensions;
  return r;
}

// The request of a packed entry point, with its per-utterance options.
inline ChainRequest packed_request(const void *x, int nbit, int n, const long long *x_offsets, int fs,
                                   const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                   const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                                   const D4COption *d4c_options, double *time_axis, double *f0, double *spectrogram,
                                   double *aperiodicity) {
  ChainRequest r(x, nbit, n, 0, nullptr, fs, opt, time_axis, f0, 0, spectrogram, aperiodicity);
  r.packed = true; r.x_offsets = x_offsets;
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options;
  return r;
}

struct ChainPlan {
  double frame_period = 0.0;            // ms, of the chain's F0 method
  std::vector<int> f_len;               // [n] frames of each utterance
  int f0_stride = 0;                    // the request's, or (f0_stride 0, packed) the largest frame count
  std::vector<int> x_len;               // packed: [n] samples of each utterance
  std::vector<long long> f_off;         // packed: [n + 1] frame offsets, f_off[n] = F
  size_t sp_row = 0, ap_row = 0;        // doubles per frame of the spectrogram / aperiodicity rows
  bool want_sp = false, want_ap = false;   // CheapTrick / D4C run (coded rows below 12 kHz have no bands: no D4C)
  StagePlan ct, d4;                        // the stage plans of CheapTrick / D4C, where they run (transform: both)
};

// Every check of an analysis chain, before anything is queued (the stage plans' included: a chain whose StoneMask or
// D4C cannot run at its fs is rejected here): EINVAL with last_error "<who>: ...", naming the first bad utterance
// where there is one.  Fills the plan that chain_f0 / chain_spectral and the drivers read.
int chain_plan(Ctx *c, const ChainRequest &r, const char *who, ChainPlan *p);
// The chain's stages for utterances [u0, u0 + m) of a planned request, enqueued on h (a lane, or the pipeline's
// context): x, time_axis, f0, sp and ap are device rows that start at utterance u0.  chain_f0: Harvest, or DIO +
// StoneMask (the F0 stage calls).  chain_spectral: one Batch of the rows for both drivers, CheapTrick into sp, then D4C
// into ap; a NULL sp or ap skips that stage.
// A packed request's slice: x, time_axis and f0 are the lane's padded rows of x_stride samples and f0_stride frames;
// sp / ap are packed rows, utterance u0 + k's frame 0 at row f_off[k] (DEVICE, [m]).
struct PackedSlice {
  int x_stride, f0_stride;
  const long long *f_off;
};
int chain_f0(WorldB200 *h, const ChainRequest &r, const ChainPlan &p, int u0, int m, const double *x, double *time_axis,
             double *f0, const PackedSlice *ps = nullptr);
int chain_spectral(WorldB200 *h, const ChainRequest &r, const ChainPlan &p, int u0, int m, const double *x,
                   const double *time_axis, const double *f0, double *sp, double *ap, const PackedSlice *ps = nullptr);
// The packed chain over utterances [c0, c1) of a planned packed request, in lane slices: x points at sample
// x_offsets[c0] (DEVICE, doubles or PCM) and the outputs at frame f_off[c0] (DEVICE, NULL sp / ap: not computed).
// The analysis runs on padded slice rows; only x is read, and only the outputs' frames [f_off[c0], f_off[c1]) written.
int packed_run(WorldB200 *h, const ChainRequest &r, const ChainPlan &p, int c0, int c1, const void *x,
               double *time_axis, double *f0, double *sp, double *ap);
// x_offsets[u] .. x_offsets[u + 1] -> padded rows: out[k][x_stride] (k < m) gets utterance k's samples, converted from
// nbit-bit PCM by pcm_to_double's rule (nbit 0: copied); x_off is DEVICE [m + 1], relative to x.  Values past an
// utterance's length are not written.
int gather_samples(Ctx *ctx, const void *x, int nbit, const long long *x_off, int m, int max_len, int x_stride,
                   double *out);

// Voice transformation (world_b200_transform_*): the analysis plan of the request (full rows, no analysis outputs;
// with spectral options each row as wide as the largest size's) and the synthesis plan of its analysis rows: lengths,
// each utterance's CheapTrick size, the factors (which modify_run applies right after the analysis) and each
// utterance's frame period, (frame_period * time_scale[u]) / 1000.0 s.  A packed request (r.packed) gets a packed
// synthesis plan: the chain's frame offsets, sample offsets from world_b200_transform_samples, every utterance at its
// CheapTrick size on rows of sp_row doubles.  transform_check makes it once per call; transform_run (device rows) and
// the host pipelines (wb_host.cu) read it.
struct TransformPlan {
  ChainPlan chain;
  SynthesisPlan syn;
};
// y_stride is not read for a packed request.
int transform_check(WorldB200 *h, const ChainRequest &r, const double *f0_scale, const double *spectral_ratio,
                    const double *time_scale, int nbit_out, void *y, int y_stride, const char *who, TransformPlan *tp);
// Utterances [u0, u0 + n) of a checked call: x and y point at utterance u0's rows (device); packed: at its first sample
// of x and of y.  cv (packed only, checked curves): DEVICE curves on the analysis frames, at utterance u0's first frame;
// each slice's frames are modified by curves_run in place of modify_run.
int transform_run(WorldB200 *h, const ChainRequest &r, const TransformPlan &tp, const void *x, int u0, int n, void *y,
                  const ModifyCurves *cv = nullptr);

}  // namespace wb
