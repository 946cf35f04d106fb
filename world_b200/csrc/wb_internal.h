// wb_internal.h -- host-side context shared by the stage drivers (not part of the public ABI).
#pragma once
#include "wb_platform.cuh"
#include "wb_block.cuh"
#include "wb_fft.cuh"
#include <string>
#include <vector>

#define WB_RNG_CHUNK 128   // draws produced by one rng_fill thread
#define WB_RNG_NJ 24       // jump tables J_k = T^(12*128*2^k): reach 2^31 draws per utterance
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
  uint32_t *rng_jump = nullptr;      // [WB_RNG_NJ][32][16] uint4
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
void rng_fill(const Ctx *ctx, const unsigned *totals_dev, unsigned *out, size_t utt_stride,
              size_t max_draws_per_utt, int n_utts);
void scan_counts(const Ctx *ctx, const unsigned *counts, const int *lens_dev, int stride,
                 const unsigned *base, unsigned *offsets, unsigned *totals, int n_utts);

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
int cheaptrick_run(Ctx *ctx, const Batch &b, double q1, int fft_size, double *spectrogram,
                   const CodecTables *coded = nullptr, double *coded_out = nullptr);
int d4c_run(Ctx *ctx, const Batch &b, int fft_size, double threshold, double *aperiodicity,
            const CodecTables *coded = nullptr, double *coded_out = nullptr);
int stonemask_run(Ctx *ctx, const Batch &b, double *refined_f0);
struct DioParams { double f0_floor, f0_ceil, channels_in_octave, frame_period, allowed_range; int speed; };
int dio_run(Ctx *ctx, const Batch &b, const DioParams &p, double *time_axis_out, double *f0_out);
struct HarvestParams { double f0_floor, f0_ceil, frame_period; };
int harvest_run(Ctx *ctx, const Batch &b, const HarvestParams &p, double *time_axis_out, double *f0_out);

}  // namespace wb
