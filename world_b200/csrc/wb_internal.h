// wb_internal.h -- host-side context shared by the stage drivers (not part of the public ABI).
#pragma once
#include "wb_platform.cuh"
#include "wb_block.cuh"
#include "wb_fft.cuh"
#include "../../include/world/dio.h"
#include "../../include/world/harvest.h"
#include "../../include/world/cheaptrick.h"
#include "../../include/world/d4c.h"
#include <string>
#include <vector>

#define WB_RNG_CHUNK 128   // draws produced by one rng_fill thread
#define WB_RNG_NJ 24       // jump tables J_k = T^(12*128*2^k), one per bit of the chunk index
// draws per utterance the tables reach (2^31): a stage whose draws would go further reports WORLD_B200_EDOMAIN
#define WB_RNG_REACH ((unsigned long long)WB_RNG_CHUNK << WB_RNG_NJ)
#define WB_RNG_WARPS 4

namespace wb {

// Bump allocator over one device allocation; stage drivers carve their scratch out of it and
// reset it when they return.  Grows (cudaMalloc) only when a request does not fit.
struct Arena {
  unsigned char *base = nullptr;
  size_t capacity = 0, used = 0;
};

// Pinned staging ring for the small host tables every stage call uploads (lengths, filter taps, index
// tables).  cudaMemcpyAsync from PAGEABLE memory first waits for the stream to drain, which would
// serialise host and device at every stage call; copies out of this ring are truly asynchronous, so the
// host keeps running ahead of the GPU.  Two halves; a half is reused only after the event recorded when
// it was left has completed.
struct Staging {
  unsigned char *base = nullptr;
  size_t half_bytes = 0, used = 0;
  int half = 0;
  void *left_event[2] = {nullptr, nullptr};   // cudaEvent_t
  bool pending[2] = {false, false};
};

// Device buffers of the host pipelines, kept between calls (cudaMalloc / cudaFree of tens of GB per call
// cost more than the uploads they serve); world_b200_trim() gives them back.
struct PoolBuf { void *p; size_t cap; bool busy; };

struct Ctx {
  int device = 0;
  wb_stream_t stream = 0;
  double2 *twiddle = nullptr;        // [WB_TW_N/2] exp(-j 2 pi k / WB_TW_N)
  double2 *twiddle_sized = nullptr;  // [WB_TW_SIZED_ENTRIES] the same values, one contiguous table per size (wb_fft.cuh)
  uint32_t *rng_jump = nullptr;      // [WB_RNG_NJ][32][16] uint4
  // Draws [0, rng_table_len) of the randn() stream, the exact uint32 sums (those below WB_RNG_REACH filled): every
  // CheapTrick, D4C and Synthesis call reads its frames' draws at their stream offsets here (rng_table_reserve)
  unsigned *rng_table = nullptr;
  size_t rng_table_len = 0;
  Arena arena;
  Staging staging;
  std::vector<PoolBuf> pool;
  size_t scratch_budget = (size_t)24 << 30;  // bytes of scratch a stage may use per chunk
  int sm_count = 132;
  int *status_dev = nullptr;         // sticky device-side error word
  std::string last_error;
};

// The CUDA current device is per thread; every extern "C" entry point that touches a context makes the
// context's device current for its own duration (a call from another thread, or a second context on another GPU
// of the same process, would otherwise allocate and launch on the caller's device) and restores the caller's.
struct DeviceGuard {
#ifndef WB_EMU
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const Ctx *c) {
    if (c && cudaGetDevice(&prev) == cudaSuccess && prev != c->device) switched = cudaSetDevice(c->device) == cudaSuccess;
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
#else
  explicit DeviceGuard(const Ctx *) {}
#endif
  DeviceGuard(const DeviceGuard &) = delete;
  DeviceGuard &operator=(const DeviceGuard &) = delete;
};

// memory helpers (wb_api.cu / emu)
int ctx_init_tables(Ctx *ctx);
unsigned char *arena_block(Ctx *ctx, size_t bytes);  // nullptr + last_error on failure
// Utterances per pass when `fit` fit the scratch budget: as few passes as possible, evenly sized
// (per-utterance kernels cost one launch latency per pass whatever its size).
inline int balanced_chunk(int n, int fit) {
  if (fit < 1) fit = 1;
  if (n <= fit) return n > 0 ? n : 1;
  const int passes = (n + fit - 1) / fit;
  return (n + passes - 1) / passes;
}
// The u in [0, n) with off[u] <= x < off[u + 1] for ascending off with off[0] <= x < off[n]: the largest u with
// off[u] <= x, so that empty entries are passed over.
WB_HD inline int packed_find(const long long *off, int n, long long x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct ArenaPlan {                                   // lay out 256-byte aligned sub-blocks
  size_t total = 0;
  size_t add(size_t bytes) { const size_t off = total; total += (bytes + 255) & ~(size_t)255; return off; }
};

void *pool_acquire(Ctx *ctx, size_t bytes);   // cached device buffer >= bytes (nullptr + last_error on failure)
void pool_release(Ctx *ctx, void *p);
void pool_trim(Ctx *ctx);                     // frees every idle pooled buffer
void *dev_malloc(Ctx *ctx, size_t bytes);
void dev_free(void *p);
int dev_memcpy_h2d(Ctx *ctx, void *dst, const void *src, size_t bytes);
int dev_memcpy_d2h(Ctx *ctx, void *dst, const void *src, size_t bytes);
int dev_memset(Ctx *ctx, void *dst, int value, size_t bytes);
int dev_sync(Ctx *ctx);
int dev_check(Ctx *ctx, const char *what);      // cudaGetLastError -> last_error

// wb_rng.cu
void rng_build_jump_tables(uint32_t *tables);
// draws [first, end) of the stream into out[0, end - first) (end <= WB_RNG_REACH)
void rng_fill(const Ctx *ctx, unsigned *out, unsigned first, unsigned end);
// The context's stream table holding at least draws [0, draws) (nullptr + last_error on failure).  The table is context
// memory like the twiddle and jump tables, outside the scratch budget: it grows (synchronise, free, allocate a little
// more than asked, fill) and never shrinks except through world_b200_trim().  Draws at and past WB_RNG_REACH are
// allocated but not generated: a call whose offsets reach them has had scan_counts flag WORLD_B200_EDOMAIN.
const unsigned *rng_table_reserve(Ctx *ctx, size_t draws);
// counts / offsets of utterance u at u * stride, or with utt_off (device, [n_utts]) at utt_off[u]
void scan_counts(const Ctx *ctx, const unsigned *counts, const int *lens_dev, int stride,
                 const unsigned *base, unsigned *offsets, unsigned *totals, int n_utts,
                 const long long *utt_off = nullptr);

// wb_multi.cu: NCCL communicator behind the C ABI (bound at run time)
struct Comm;
int comm_unique_id(unsigned char *id128, std::string *err);
int comm_create(int n_ranks, int rank, const unsigned char *id128, Comm **out, std::string *err);
void comm_destroy(Comm *c);
int comm_ranks(const Comm *c);
int comm_rank(const Comm *c);
#ifndef WB_EMU
int comm_gather_rows(Comm *c, double *full, size_t row_elems, size_t rows_per_rank, size_t row0, size_t rows,
                     cudaEvent_t after, std::string *err);
int comm_gather_rows_multi(Comm *c, int n_arrays, double *const *full, const size_t *row_elems, size_t rows_per_rank,
                           size_t row0, size_t rows, cudaEvent_t after, std::string *err);
int comm_join(Comm *c, cudaStream_t s, std::string *err);
// peer-to-peer push of finished rows over CUDA IPC mappings (copy engines); prepare: 0 usable, 1 not usable, 2 error
int comm_p2p_prepare(Comm *c, int n_arrays, double *const *full, std::string *err);
int comm_p2p_push(Comm *c, int n_arrays, const size_t *row_elems, size_t rows_per_rank, size_t row0, size_t rows,
                  cudaEvent_t after, std::string *err);
int comm_p2p_finish(Comm *c, cudaStream_t s, std::string *err);
#endif

// Device-resident batch: N utterances, padded rows.
struct Batch {
  const double *x;        // [n][x_stride]
  const int *x_len;       // [n] device
  int n, x_stride, fs;
  const double *time_axis;  // [n][f_stride]
  const double *f0;         // [n][f_stride]
  const int *f_len;         // [n] device
  int f_stride;
  int max_x_len, max_f_len;  // host-known maxima
  const int *l1_host = nullptr;  // [n] host: frames on the 1 ms grid (Harvest only)
  const int *x_len_host = nullptr;  // [n] host copy of x_len, or nullptr = every row is full (DIO only)
  // CheapTrick / D4C output rows: [n] device frame offsets (packed rows, utterance u's frame i at row f_off[u] + i), or
  // nullptr = padded rows (u * f_stride + i)
  const long long *f_off = nullptr;
  // Packed inputs (the packed stage calls): [n] device sample offsets, utterance u's samples at x + x_off[u].  With them
  // f_off ([n + 1], from 0) also places the input frames -- time_axis / f0 at f_off[u] + i -- and the stages' per-frame
  // scratch follows the packed frames; f_off_host is its host copy.  nullptr = padded inputs (x_stride / f_stride).
  const long long *x_off = nullptr;
  const long long *f_off_host = nullptr;
};

// stage drivers (each: enqueue on ctx->stream, return 0 / error code)
// Coded output straight from the frame kernels (SURVEY.md 8 row f2): the tables of CodeSpectralEnvelope /
// CodeAperiodicity (codec.cpp:161-181, :228-238), host made by wb_codec.cu, ride along to the stage drivers; with
// them the frame kernels write the coded row instead of the fft_size/2+1 bins and the full row never reaches HBM.
struct CodecTables {
  std::vector<int> idx; std::vector<double> frac; std::vector<double2> weight;
  int dims = 0, lg_half = 0;   // coded values per frame; log2(fft_size / 2) (spectral envelope only)
  double norm = 1.0;           // sqrt(fft_size / 2)
};
int codec_sp_tables(Ctx *ctx, int fs, int fft_size, int number_of_dimensions, CodecTables *t);
int codec_ap_tables(Ctx *ctx, int fs, int fft_size, CodecTables *t);   // t->dims = 0 below 12 kHz
// The decode half of the codec for a driver that lays out its own scratch (Synthesis from coded rows decodes chunk
// by chunk into its own block): the tables world_b200_decode_*_batch build, and the launch of their kernels over
// tables, lengths (f_len, n_utts entries, largest max_f) and rows already on the device.
int codec_decode_sp_tables(Ctx *ctx, int fs, int fft_size, int number_of_dimensions, CodecTables *t);
void codec_decode_ap_tables(int fs, int fft_size, CodecTables *t);    // t->dims = GetNumberOfAperiodicities(fs)
// list: the n_utts utterances to decode are list[0 .. n_utts) of the rows (NULL: 0 .. n_utts); out_row: doubles per
// decoded frame row (>= fft_size / 2 + 1).
struct CodecDeviceTables { const int *idx; const double *frac; const double2 *weight; };
void codec_decode_launch(Ctx *ctx, bool spectral_envelope, const CodecTables &t, const CodecDeviceTables &d,
                         int fft_size, const int *f_len, int n_utts, int f_stride, int max_f, const double *in,
                         double *out, const int *list = nullptr, int out_row = 0);
// The same over packed rows, one CTA per frame: utterance u's frame i is row f_off[u] + i of both in and out (device,
// [n + 1]; f_len: device, [n]).  The launch decodes `frames` frames: entry j of list (list_n entries; NULL: utterance j)
// owns frames cum[j] .. cum[j + 1] - 1 of the grid (cum: device, [list_n + 1]).
void codec_decode_packed_launch(Ctx *ctx, bool spectral_envelope, const CodecTables &t, const CodecDeviceTables &d,
                                int fft_size, const int *f_len, const long long *f_off, const int *list, int list_n,
                                const long long *cum, long long frames, const double *in, double *out, int out_row);
// wb_synthesis.cu: F0 scaling and spectral stretch (the reference demo's ParameterModification, test.cpp:221-258).
// The interp1 segment and weight of each output bin depend only on (ratio, fft_size, fs), so they are planned on the
// host once per distinct (ratio, fft_size); the tail rule (bins >= c copy bin c-1 when ratio < 1) is folded into the
// table.
struct ModifyPlan {
  std::vector<double> scale;   // [n_utts] f0 factor of each utterance; empty: f0 is not scaled
  std::vector<int> table;      // [n_utts] stretch table of each utterance; empty: the envelope is not stretched
  std::vector<int> idx;        // [sum of tbins] a = k - 1 of interp1's segment (the kernel reads L[a], L[a + 1])
  std::vector<double> frac;    // [sum of tbins] s = (xi - x[a]) / (x[a + 1] - x[a])
  std::vector<int> tbins, toff;   // [n_tables] bins of each table (its fft_size / 2 + 1) and its first entry
  int n_tables = 0, bins = 0;     // bins: the largest table's
  size_t device_bytes(int n) const;   // arena bytes of one pass of n utterances: tables, factors, table indices
};
// Checks every factor (finite, > 0; a ratio below 1 must keep c = (int)(fft_size / 2.0 * ratio) >= 1) and builds the
// plan; EINVAL with last_error "<who>: ..." naming the first bad utterance.  Either array may be null.  fft_sizes:
// utterance u's size (checked by the caller), or NULL: fft_size (checked here) for every utterance.
int modify_plan(Ctx *ctx, const char *who, int n_utts, int fft_size, int fs, const double *f0_scale,
                const double *spectral_ratio, ModifyPlan *plan, const int *fft_sizes = nullptr);
// Plan entries [u0, u0 + n) in device memory (layout of device_bytes); the copies are enqueued on ctx->stream.
struct ModifyDevice { const double *scale; const int *table; const int *idx; const double *frac; const int *tbins, *toff; };
int modify_upload(Ctx *ctx, const ModifyPlan &plan, int u0, int n, unsigned char *blk, ModifyDevice *d);
// f0_out[u][i] = f0_in[u][i] * scale[u] for i < f_len[u] (f0_out may alias f0_in).  f_off (device, [n_utts + 1]):
// packed rows, utterance u's frame i at f_off[u] + i; NULL: padded rows of f_stride.
void modify_f0_launch(Ctx *ctx, const ModifyDevice &d, const int *f_len, int n_utts, int f_stride, int max_f,
                      const double *f0_in, double *f0_out, const long long *f_off = nullptr);
// the envelope rows [n][f_stride][row] stretched in place, frames < f_len[u], the first bins of the utterance's table
// of each row (max_bins: the plan's largest); f_off as for modify_f0_launch
void modify_stretch_launch(Ctx *ctx, const ModifyDevice &d, int row, int max_bins, const int *f_len, int n_utts,
                           int f_stride, int max_f, double *spectrogram, const long long *f_off = nullptr);

// Both halves of the plan on the device rows of its utterances [u0, u0 + n_utts) in place (f0 [n][f0_stride],
// spectrogram [n][f0_stride][row], row >= plan.bins; host lengths), frames < f0_lengths[u]: world_b200_modify_batch's
// launches.
// f_offsets (host, [n_utts + 1]): packed rows, utterance u's frame i at row f_offsets[u] + i (f0_stride is not read).
int modify_run(Ctx *ctx, const ModifyPlan &plan, int u0, int n_utts, const int *f0_lengths, int f0_stride, int row,
               double *f0, double *spectrogram, const long long *f_offsets = nullptr);

// Pitch and formant curves: one f0 factor and one spectral ratio per frame, laid out as the frames' rows (padded
// [n][f_stride], or packed [F] at the frame offsets).  Either may be null (that half is not modified).
struct ModifyCurves { const double *f0 = nullptr, *ratio = nullptr; };
// modify_plan's rule for every frame < f_len[u] of each curve (ratio: at fft_sizes[u]), on DEVICE curves: one check
// kernel and one read-back, so ctx->stream is synchronised.  Host lengths, sizes and offsets (f_off [n_utts + 1]: packed
// rows; null: padded rows of f_stride).  EINVAL with last_error "<who>: f0_curve[i] = v (utterance u, frame f) ..." for
// the first bad frame of the first bad curve; nothing is modified.
int curves_check(Ctx *ctx, const char *who, const ModifyCurves &cv, int n_utts, const int *f_len, int f_stride,
                 const long long *f_off, const int *fft_sizes);
// The same rule on HOST curves
int curves_check_host(Ctx *ctx, const char *who, const ModifyCurves &cv, int n_utts, const int *f_len, int f_stride,
                      const long long *f_off, const int *fft_sizes);
// Both halves on the device rows in place (checked curves; the layout of curves_check, row doubles per envelope frame):
// modify_curve_f0_kernel and modify_curve_stretch_kernel, enqueued on ctx->stream.
int curves_run(Ctx *ctx, const ModifyCurves &cv, int n_utts, const int *f_len, int f_stride, const long long *f_off,
               const int *fft_sizes, int fs, int row, double *f0, double *spectrogram);

// out[u] = lengths[u] (NULL: stride) for u < n; EINVAL "<who>: <rows>_lengths[u] = v is outside [least, <rows>_stride =
// stride] (utterance u)" for the first one outside
int row_lengths(Ctx *ctx, const char *who, const char *rows, const int *lengths, int n, int stride, int least,
                std::vector<int> *out);

// wb_synthesis.cu: the Synthesis driver, shared by the device entry points, the host pipeline (wb_host.cu) and voice
// transformation (wb_api.cu): one checked plan per call, then synthesis_run over the rows of each chunk or slice.
// What a synthesis call receives: f0 [n][f0_stride], the envelope rows sp / ap (spectrogram / aperiodicity
// [n][f0_stride][bins], or with `coded` [n][f0_stride][dims] / [GetNumberOfAperiodicities(fs)] coded rows) and y
// [n][y_stride] (doubles for nbit 0, int16 for nbit 16).  NULL lengths: full rows.  NULL factors: no modification.
// per_utt: utterance u is synthesised at fft_sizes[u] (fft_size is not read), and full rows hold row_stride doubles
// per frame, of which utterance u reads fft_sizes[u] / 2 + 1.
struct SynthesisRequest {   // brace-initialised in field order up to nbit
  const double *f0;
  const int *f0_lengths;
  int n, f0_stride;
  const double *sp, *ap;
  int fft_size;
  double frame_period;   // ms
  int fs;
  const int *y_lengths;
  int y_stride;
  void *y;
  int nbit;
  bool coded = false;
  int dims = 0;          // coded: number_of_dimensions
  const double *f0_scale = nullptr, *spectral_ratio = nullptr;
  // transform: f0 / sp / ap are the call's own analysis rows, not given here, and fp [n] holds each utterance's frame
  // period (s)
  bool transform = false;
  const double *fp = nullptr;
  bool per_utt = false;
  const int *fft_sizes = nullptr;
  int row_stride = 0;
  // packed (per_utt): utterance u is frames [f_offsets[u], f_offsets[u + 1]) of f0 / sp / ap and samples
  // [y_offsets[u], y_offsets[u + 1]) of y (host arrays, n + 1 entries); f0_lengths, y_lengths and the strides are not
  // read, and row_stride 0 is the largest fft_sizes[u] / 2 + 1
  const long long *f_offsets = nullptr, *y_offsets = nullptr;
};
// Everything synthesis_run reads besides the rows, made once per call and const afterwards.
// Sizes: every per-size member has one entry per distinct fft_size of the call, in order of first appearance (one
// entry for a one-size call).
struct SynthesisPlan {
  int n = 0, f0_stride = 0, y_stride = 0, fs = 0, nbit = 0;
  int fft_size = 0;                 // the largest fft_size of the call: responses and decoded rows are laid out by it
  int row = 0;                      // doubles per full (or decoded) envelope frame row
  double frame_period = 0.0;        // ms
  std::vector<int> f_len, y_len;    // [n]
  std::vector<int> size;            // [n] index of each utterance's fft_size in sizes
  std::vector<int> sizes;           // the distinct fft_sizes
  bool coded = false;
  std::vector<CodecTables> tsp, tap;   // per size, coded: the decode tables (tap dims 0 below 12 kHz: no rows)
  int dims = 0, n_ap = 0;              // coded values per envelope / aperiodicity frame
  // f0_scale or spectral_ratio given.  synthesis_run applies it to coded rows, as it decodes them; full rows are their
  // producer's to modify (transform runs modify_run on its analysis rows).
  bool modify = false;
  ModifyPlan mod;
  std::vector<double> fp;           // [n] frame period (s) of each utterance, or empty: frame_period / 1000.0 for all
  std::vector<std::vector<double>> dc_remover;   // per size: [fft_size] GetDCRemover (synthesis.cpp:319-333)
  // packed rows: [n + 1] frame and sample offsets (f_len / y_len derived from them); empty: padded rows
  std::vector<long long> f_off, y_off;
  bool packed() const { return !f_off.empty(); }
};
// Every check of a synthesis call before anything is queued, in this order: the pointers, n, fs and frame_period;
// nbit; fft_size (per_utt: each utterance's, a power of two in [16, 4096]); per_utt full rows: row_stride against each
// utterance's bins; the coded decode tables (per_utt: number_of_dimensions in [1, fft_sizes[u] / 2]); the factors
// (modify_plan); each utterance's f0 and y lengths (2 .. stride; packed: the offsets start at 0 and give each
// utterance 2 .. INT_MAX frames and samples).  EINVAL with last_error "<who>: ...", naming the first bad utterance where
// there is one.
int synthesis_plan(Ctx *ctx, const SynthesisRequest &r, const char *who, SynthesisPlan *p);
// Per-utterance scratch of synthesis_run for rows whose longest y_length is max_y; fit(nominal_cap) utterances make one
// pass when no utterance has more than 1,200 pulses per second.
// A packed pass holds each utterance's own scratch instead: packed_utt(y_len, f_len, cap) bytes for an utterance of
// y_len samples and f_len frames with room for cap pulses (cap_of(y_len) when it has at most 1,200 per second), plus
// packed_pass bytes per pass.
struct SynthesisSizing {
  SynthesisSizing(const Ctx *ctx, const SynthesisPlan &p, int max_y);
  size_t per_utt(int cap) const;
  int fit(int cap) const;
  int cap_of(int y_len) const;
  size_t packed_utt(int y_len, int f_len, int cap) const;
  size_t packed_pass() const;
  int fft_size, y_stride, nominal_cap, fs;   // fft_size: the plan's largest, the stride of each response
  size_t decoded_per_utt, max_draws, decoded_per_frame;
  double budget;
};
// The rows of utterances [u0, u0 + m) of a planned call: device pointers at utterance u0 (packed: at its first frame
// and first sample), laid out as the request's
// (sp / ap: full or coded rows, as the plan says; coded ap is not read below 12 kHz, where there are no bands).
struct SynthesisRows {
  const double *f0, *sp, *ap;
  void *y;
};
// Enqueues Synthesis of the plan's utterances [u0, u0 + m) on ctx->stream, in passes that fit the scratch budget, each
// with one read-back of its pulse counts.  With coded rows and factors, each pass synthesises from a scaled copy of its
// f0 rows and stretches its decoded envelope block right after the decode.
int synthesis_run(Ctx *ctx, const SynthesisPlan &p, int u0, int m, const SynthesisRows &rows);

// The CheapTrick, D4C and StoneMask stages: one checked plan per call (a stage entry point, or an analysis chain), then
// a run over the rows of each batch, slice or chunk.  What a stage call receives besides its device rows: n utterances
// of x_stride samples and f0_stride frames (NULL lengths: full rows) at fs, and the stage's option -- one (per_utt
// false) or one per utterance.  CheapTrick takes ct; D4C takes its fft_size and d4c.  coded: the rows take dims
// (CheapTrick) or GetNumberOfAperiodicities(fs) (D4C) coded values per frame.  row_stride: doubles per full row, at
// least every utterance's fft_size / 2 + 1 (0: the one option's fft_size / 2 + 1).
enum StageKind { STAGE_CHEAPTRICK, STAGE_D4C, STAGE_STONEMASK };
struct StageRequest {   // brace-initialised in field order up to f0_stride
  StageKind stage;
  int n, x_stride;
  const int *x_lengths;
  int fs;
  const int *f0_lengths;
  int f0_stride;
  bool per_utt = false;
  const CheapTrickOption *ct = nullptr;
  const int *fft_size = nullptr;
  const D4COption *d4c = nullptr;
  bool coded = false;
  int dims = 0;
  int row_stride = 0;
  // packed (per_utt): utterance u is samples [x_offsets[u], x_offsets[u + 1]) and frames [f_offsets[u], f_offsets[u + 1])
  // (host arrays, n + 1 entries); the lengths and strides are not read, and row_stride 0 is the largest
  // fft_size[u] / 2 + 1
  const long long *x_offsets = nullptr, *f_offsets = nullptr;
};
// Everything a stage run reads besides the rows, made once per call and const afterwards.
struct StagePlan {
  std::vector<int> x_len, f_len;    // [n]
  std::vector<int> fft_size;        // [n] CheapTrick / D4C
  std::vector<double> q;            // [n] q1 (CheapTrick) or threshold (D4C)
  bool coded = false;
  std::vector<int> table;           // [n] coded: the utterance's entry of tables
  std::vector<CodecTables> tables;  // coded: one per distinct fft_size, in order of first appearance
  int row = 0;                      // doubles per full output row
  bool nothing = false;             // coded D4C below 12 kHz: no bands, nothing to write (a NULL output is allowed)
  std::vector<long long> x_off, f_off;   // packed: the request's offsets [n + 1]; empty: padded rows
};
// Every check of a stage call before anything is queued, in this order: n and fs; the stage's sampling-rate limits
// (StoneMask: fs <= 48 kHz; D4C: its transforms within the on-chip FFT); each option (CheapTrick: fft_size a power of
// two in [16, 8192], q1 finite; D4C: fft_size >= 4, threshold finite); row_stride; the codec tables of each distinct
// fft_size; each utterance's x and f0 lengths (1 .. x_stride, 0 .. f0_stride; packed: the offsets start at 0 and give
// each utterance 1 .. INT_MAX samples and 0 .. INT_MAX frames).  EINVAL with last_error "<stage>: ...", naming the first
// bad utterance where there is one.
int stage_plan(Ctx *ctx, const StageRequest &r, StagePlan *p);
// The rule of packed offsets: off (host, n + 1) starts at 0 and every utterance spans least .. INT_MAX `unit`, filling
// len [n]; "" when they are good, else the broken rule naming the first bad utterance.
std::string packed_lengths(const char *name, const char *unit, int n, const long long *off, int least,
                           std::vector<int> *len);
// Scratch of the packed stage runs, by which the packed stage calls cut their utterances into chunks of at most the
// scratch budget: per packed frame, CheapTrick's draw count and offset, and D4C's two counts, two offsets, selected
// flag, frame-list entry and frame utterance (ct_launch and d4c_run check their layouts against these); per utterance,
// their per-utterance arrays (totals, group indices, offsets, options); per chunk, the arrays' 256-byte alignment and
// the codec tables.
constexpr size_t WB_CT_FRAME_BYTES = 2 * sizeof(unsigned);
constexpr size_t WB_D4C_FRAME_BYTES = 4 * sizeof(unsigned) + 1 + 2 * sizeof(int);
constexpr size_t WB_STAGE_FRAME_BYTES = WB_CT_FRAME_BYTES > WB_D4C_FRAME_BYTES ? WB_CT_FRAME_BYTES : WB_D4C_FRAME_BYTES;
constexpr size_t WB_STAGE_UTT_BYTES = 64;
constexpr size_t WB_STAGE_CHUNK_BYTES = (size_t)1 << 20;
// The stage over batch b, whose rows are the plan's utterances [u0, u0 + b.n) (its lengths uploaded from the plan's).
// CheapTrick runs one launch sequence per distinct (fft_size, q1) among them, in order of first appearance; D4C one
// launch sequence, with per-utterance device arrays when their options differ.  out: full or coded rows, as planned.
int cheaptrick_run(Ctx *ctx, const StagePlan &plan, const Batch &b, int u0, double *out);
int d4c_run(Ctx *ctx, const StagePlan &plan, const Batch &b, int u0, double *out);
int stonemask_run(Ctx *ctx, const Batch &b, double *refined_f0);
// the stages' sampling-rate limits (stage_plan): D4C's transforms and StoneMask's largest window fit the on-chip FFT
bool d4c_fits(int fs);
bool stonemask_fits(int fs);
// The F0 estimators (wb_harvest.cu, wb_dio.cu) take the public options.  Per utterance (per_utt: opts[u] is utterance
// u's, else opts[0] serves all), the F0 range may differ, frame_period (DIO: and speed) may not.  *_plan checks that
// frame_period (and speed) against the batch's, then groups the utterances by range and builds each group's band list
// (wb_f0common.cuh): 3 (EINVAL) + last_error naming the first bad utterance.  It queues nothing, so a call runs it
// before its lengths are uploaded, and *_run takes its groups.
struct RangeGroups;
int harvest_plan(Ctx *ctx, int fs, const HarvestOption *opts, int n, bool per_utt, double frame_period,
                 RangeGroups *groups);
int harvest_run(Ctx *ctx, const Batch &b, double frame_period, const RangeGroups &groups, double *time_axis_out,
                double *f0_out);
int dio_plan(Ctx *ctx, int fs, const DioOption *opts, int n, bool per_utt, double frame_period, int speed,
             RangeGroups *groups);
int dio_run(Ctx *ctx, const Batch &b, const DioOption *opts, bool per_utt, const RangeGroups &groups,
            double *time_axis_out, double *f0_out);

}  // namespace wb
