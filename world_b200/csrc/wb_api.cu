// wb_api.cu -- context, scratch arena and the extern "C" ABI declared in include/world_b200.h,
// plus the legacy single-utterance entry points of include/world/*.h implemented as n_utts = 1
// batches (reference boundary: src/world/{dio,harvest,stonemask,cheaptrick,d4c}.h).
#include "wb_internal.h"
#include "../../include/world_b200.h"
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <vector>
#include <string>

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

unsigned long long g_launches = 0;
int g_prof_on = 0;

#ifndef WB_EMU
namespace {
struct ProfRec { const char *name; cudaEvent_t a, b; };
std::vector<ProfRec> g_prof;
std::vector<cudaEvent_t> g_prof_pool;
cudaEvent_t prof_event() {
  cudaEvent_t e;
  if (!g_prof_pool.empty()) { e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEventCreate(&e);
  return e;
}
}  // namespace
void prof_begin(const char *name, cudaStream_t s) {
  ProfRec r; r.name = name; r.a = prof_event(); r.b = prof_event();
  cudaEventRecord(r.a, s);
  g_prof.push_back(r);
}
void prof_end(cudaStream_t s) { cudaEventRecord(g_prof.back().b, s); }
#endif

#ifndef WB_EMU
static int cuda_fail(Ctx *ctx, cudaError_t e, const char *what) {
  ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  return WORLD_B200_ECUDA;
}
#define WB_CUDA(ctx, call, what)                                \
  do {                                                          \
    cudaError_t e_ = (call);                                    \
    if (e_ != cudaSuccess) return cuda_fail((ctx), e_, (what)); \
  } while (0)
#endif

int dev_check(Ctx *ctx, const char *what) {
#ifndef WB_EMU
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(ctx, e, what);
#else
  (void)ctx; (void)what;
#endif
  return 0;
}

int dev_sync(Ctx *ctx) {
#ifndef WB_EMU
  WB_CUDA(ctx, cudaStreamSynchronize(ctx->stream), "stream synchronize");
#else
  (void)ctx;
#endif
  return 0;
}

#ifndef WB_EMU
// Region of `bytes` in the pinned staging ring (nullptr: too large, or no ring -- caller copies directly).
static unsigned char *staging_take(Ctx *ctx, size_t bytes) {
  Staging &st = ctx->staging;
  if (!st.base) {
    const size_t half = (size_t)8 << 20;
    if (cudaHostAlloc((void **)&st.base, 2 * half, cudaHostAllocDefault) != cudaSuccess) { st.base = nullptr; cudaGetLastError(); return nullptr; }
    st.half_bytes = half;
    for (int i = 0; i < 2; ++i) {
      cudaEvent_t e;
      cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
      st.left_event[i] = e;
    }
  }
  const size_t need = (bytes + 63) & ~(size_t)63;
  if (need > st.half_bytes) return nullptr;
  if (st.used + need > st.half_bytes) {
    // leave this half: everything copied out of it so far is ordered before this event
    cudaEventRecord((cudaEvent_t)st.left_event[st.half], ctx->stream);
    st.pending[st.half] = true;
    st.half ^= 1;
    st.used = 0;
    if (st.pending[st.half]) { cudaEventSynchronize((cudaEvent_t)st.left_event[st.half]); st.pending[st.half] = false; }
  }
  unsigned char *p = st.base + (size_t)st.half * st.half_bytes + st.used;
  st.used += need;
  return p;
}
#endif

int dev_memcpy_h2d(Ctx *ctx, void *dst, const void *src, size_t bytes) {
  if (bytes == 0) return 0;
#ifndef WB_EMU
  if (unsigned char *stage = staging_take(ctx, bytes)) {
    memcpy(stage, src, bytes);
    src = stage;
  }
  WB_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream), "memcpy h2d");
#else
  (void)ctx; memcpy(dst, src, bytes);
#endif
  return 0;
}

int dev_memcpy_d2h(Ctx *ctx, void *dst, const void *src, size_t bytes) {
  if (bytes == 0) return 0;
#ifndef WB_EMU
  WB_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream), "memcpy d2h");
#else
  (void)ctx; memcpy(dst, src, bytes);
#endif
  return 0;
}

int dev_memset(Ctx *ctx, void *dst, int value, size_t bytes) {
  if (bytes == 0) return 0;
#ifndef WB_EMU
  WB_CUDA(ctx, cudaMemsetAsync(dst, value, bytes, ctx->stream), "memset");
#else
  (void)ctx; memset(dst, value, bytes);
#endif
  return 0;
}

void pool_trim(Ctx *ctx);

void *dev_malloc(Ctx *ctx, size_t bytes) {
  void *p = nullptr;
#ifndef WB_EMU
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess && ctx && !ctx->pool.empty()) {
    // idle pipeline buffers can hold tens of GB: give them back and try once more before reporting ENOMEM
    cudaGetLastError();
    cudaStreamSynchronize(ctx->stream);
    pool_trim(ctx);
    e = cudaMalloc(&p, bytes);
  }
  if (e != cudaSuccess) {
    cuda_fail(ctx, e, "cudaMalloc");
    cudaGetLastError();
    return nullptr;
  }
#else
  (void)ctx;
  p = malloc(bytes);
#endif
  return p;
}

void dev_free(void *p) {
  if (!p) return;
#ifndef WB_EMU
  cudaFree(p);
#else
  free(p);
#endif
}

void pool_trim(Ctx *ctx) {
  std::vector<PoolBuf> keep;
  for (auto &b : ctx->pool) {
    if (b.busy) keep.push_back(b);
    else dev_free(b.p);
  }
  ctx->pool.swap(keep);
}

void *pool_acquire(Ctx *ctx, size_t bytes) {
  if (bytes == 0) bytes = 256;
  int best = -1;
  for (int i = 0; i < (int)ctx->pool.size(); ++i) {
    const PoolBuf &b = ctx->pool[i];
    if (b.busy || b.cap < bytes || b.cap > bytes + bytes / 2 + ((size_t)1 << 20)) continue;
    if (best < 0 || b.cap < ctx->pool[best].cap) best = i;
  }
  if (best >= 0) { ctx->pool[best].busy = true; return ctx->pool[best].p; }
  void *p = dev_malloc(ctx, bytes);   // trims the idle pooled buffers itself when the device is full
  if (!p) return nullptr;
  ctx->pool.push_back(PoolBuf{p, bytes, true});
  return p;
}

void pool_release(Ctx *ctx, void *p) {
  if (!p) return;
  for (auto &b : ctx->pool)
    if (b.p == p) { b.busy = false; return; }
  dev_free(p);
}

// One block of `bytes` device scratch, valid until the next arena_block() call on this
// context.  Stage drivers lay out their scratch with ArenaPlan and ask for the total; the block
// only grows (sync + free + cudaMalloc), so steady-state calls allocate nothing.
unsigned char *arena_block(Ctx *ctx, size_t bytes) {
  Arena &a = ctx->arena;
  if (bytes > a.capacity) {
    dev_sync(ctx);
    dev_free(a.base);
    a.base = nullptr;
    a.capacity = 0;
    const size_t want = bytes + (bytes >> 4) + (1 << 20);
    a.base = (unsigned char *)dev_malloc(ctx, want);
    if (!a.base) return nullptr;
    a.capacity = want;
  }
  a.used = bytes;
  return a.base;
}

int ctx_init_tables(Ctx *ctx) {
  // twiddles in long double so that every entry is correctly rounded
  std::vector<double2> tw(WB_TW_N / 2);
  const long double two_pi = 6.283185307179586476925286766559005768L;
  for (int k = 0; k < WB_TW_N / 2; ++k) {
    const long double a = two_pi * (long double)k / (long double)WB_TW_N;
    tw[k].x = (double)cosl(a);
    tw[k].y = (double)(-sinl(a));
  }
  std::vector<double2> tw_sized(WB_TW_SIZED_ENTRIES);
  for (int lg = 1; lg <= WB_TW_LOG2; ++lg)
    for (int n = 0; n < (1 << (lg - 1)); ++n) tw_sized[tw_sized_offset(lg) + n] = tw[n << (WB_TW_LOG2 - lg)];
  ctx->twiddle = (double2 *)dev_malloc(ctx, tw.size() * sizeof(double2));
  ctx->twiddle_sized = (double2 *)dev_malloc(ctx, tw_sized.size() * sizeof(double2));
  if (!ctx->twiddle || !ctx->twiddle_sized) return WORLD_B200_ENOMEM;
  std::vector<uint32_t> jump((size_t)WB_RNG_NJ * 32 * 16 * 4);
  rng_build_jump_tables(jump.data());
  ctx->rng_jump = (uint32_t *)dev_malloc(ctx, jump.size() * 4);
  ctx->status_dev = (int *)dev_malloc(ctx, sizeof(int));
  if (!ctx->rng_jump || !ctx->status_dev) return WORLD_B200_ENOMEM;
  int rc = dev_memcpy_h2d(ctx, ctx->twiddle, tw.data(), tw.size() * sizeof(double2));
  if (!rc) rc = dev_memcpy_h2d(ctx, ctx->twiddle_sized, tw_sized.data(), tw_sized.size() * sizeof(double2));
  if (!rc) rc = dev_memcpy_h2d(ctx, ctx->rng_jump, jump.data(), jump.size() * 4);
  if (!rc) rc = dev_memset(ctx, ctx->status_dev, 0, sizeof(int));
  if (!rc) rc = dev_sync(ctx);
  return rc;
}

}  // namespace wb

using namespace wb;

// ------------------------------------------------------------------------------------------
static int upload_lengths(WorldB200 *h, int n, int x_stride, const int *x_lengths, int f_stride,
                          const int *f_lengths, Batch *b) {
  Ctx *ctx = &h->c;
  if ((size_t)2 * n > h->lens_cap) {
    dev_sync(ctx);
    dev_free(h->lens_dev);
    h->lens_cap = (size_t)2 * n + 64;
    h->lens_dev = (int *)dev_malloc(ctx, h->lens_cap * sizeof(int));
    if (!h->lens_dev) { h->lens_cap = 0; return WORLD_B200_ENOMEM; }
  }
  std::vector<int> tmp((size_t)2 * n);
  int mx = 0, mf = 0;
  for (int i = 0; i < n; ++i) {
    const int xl = x_lengths ? x_lengths[i] : x_stride;
    const int fl = f_lengths ? f_lengths[i] : f_stride;
    if (xl < 1 || xl > x_stride || fl < 0 || fl > f_stride) {
      ctx->last_error = "utterance length outside its padded row";
      return WORLD_B200_EINVAL;
    }
    tmp[i] = xl; tmp[n + i] = fl;
    if (xl > mx) mx = xl;
    if (fl > mf) mf = fl;
  }
  // the previous call's kernels may still read lens_dev: same stream, so ordering is preserved
  int rc = dev_memcpy_h2d(ctx, h->lens_dev, tmp.data(), tmp.size() * sizeof(int));
  if (rc) return rc;
#ifndef WB_EMU
  // tmp is pageable: cudaMemcpyAsync has staged it before returning
#endif
  b->x_len = h->lens_dev; b->f_len = h->lens_dev + n;
  b->max_x_len = mx; b->max_f_len = mf;
  return 0;
}

static int frames_for(int fs, int x_length, double frame_period) {
  return static_cast<int>(1000.0 * x_length / fs / frame_period) + 1;
}

namespace wb {

// Per-utterance options: one frame_period for the whole batch; with ranges (fs > 0) also every utterance's F0 range
// against the on-chip limits, up front, so that a chain cut into slices or chunks names the batch's first bad utterance.
int check_harvest_options(Ctx *c, const HarvestOption *opts, int n, double frame_period, int fs) {
  for (int u = 0; u < n; ++u)
    if (!(opts[u].frame_period == frame_period)) {
      c->last_error = "harvest options: frame_period differs from the batch's (utterance " + std::to_string(u) + ")";
      return WORLD_B200_EINVAL;
    }
  if (fs <= 0 || n <= 0) return 0;
  std::vector<HarvestParams> p(n);
  for (int u = 0; u < n; ++u) p[u] = {opts[u].f0_floor, opts[u].f0_ceil, opts[u].frame_period};
  return harvest_check_options(c, fs, p.data(), n);
}

// The same for DIO: one frame_period and one speed for the whole batch (they fix the decimation ratio, the low-cut
// filter and the frame grid); with fs > 0 also every utterance's band list against the on-chip limits.
int check_dio_options(Ctx *c, const DioOption *opts, int n, double frame_period, int speed, int fs) {
  for (int u = 0; u < n; ++u) {
    const char *what = !(opts[u].frame_period == frame_period) ? "frame_period" : (opts[u].speed != speed ? "speed" : nullptr);
    if (what) {
      c->last_error = std::string("dio options: ") + what + " differs from the batch's (utterance " + std::to_string(u) + ")";
      return WORLD_B200_EINVAL;
    }
  }
  if (fs <= 0 || n <= 0) return 0;
  std::vector<DioParams> p(n);
  for (int u = 0; u < n; ++u)
    p[u] = {opts[u].f0_floor, opts[u].f0_ceil, opts[u].channels_in_octave, opts[u].frame_period, opts[u].allowed_range,
            opts[u].speed};
  return dio_check_options(c, fs, p.data(), n);
}

// Per-utterance F0 options of a chain (harvest_options or dio_options, at most one): they must belong to the chain's
// f0_method and pass check_*_options for the whole batch before a slice or chunk is queued.  `who` prefixes the error.
int check_chain_f0_options(Ctx *c, const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                           const DioOption *dio_options, int n, int fs, const char *who) {
  if (harvest_options && dio_options) {
    c->last_error = std::string(who) + ": per-utterance options of both F0 methods";
    return WORLD_B200_EINVAL;
  }
  if (harvest_options) {
    if (opt->f0_method != WORLD_B200_F0_HARVEST) {
      c->last_error = std::string(who) + ": per-utterance Harvest options need f0_method == WORLD_B200_F0_HARVEST";
      return WORLD_B200_EINVAL;
    }
    return check_harvest_options(c, harvest_options, n, opt->harvest.frame_period, fs);
  }
  if (dio_options) {
    if (opt->f0_method != WORLD_B200_F0_DIO_STONEMASK) {
      c->last_error = std::string(who) + ": per-utterance DIO options need f0_method == WORLD_B200_F0_DIO_STONEMASK";
      return WORLD_B200_EINVAL;
    }
    return check_dio_options(c, dio_options, n, opt->dio.frame_period, opt->dio.speed, fs);
  }
  return 0;
}

// The F0 stage of a chain on m utterances: Harvest, or DIO + StoneMask.  harvest_options / dio_options: nullptr (the
// chain's own option) or the options of these m utterances, checked by check_chain_f0_options.
int run_f0_stage(WorldB200 *h, const double *x, int m, int x_stride, const int *x_lengths, int fs,
                 const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options, const DioOption *dio_options,
                 const int *f0_lengths, double *time_axis, double *f0, int f0_stride) {
  if (opt->f0_method == WORLD_B200_F0_HARVEST)
    return harvest_options
               ? world_b200_harvest_batch_options(h, x, m, x_stride, x_lengths, fs, harvest_options, time_axis, f0, f0_stride)
               : world_b200_harvest_batch(h, x, m, x_stride, x_lengths, fs, &opt->harvest, time_axis, f0, f0_stride);
  int rc = dio_options
               ? world_b200_dio_batch_options(h, x, m, x_stride, x_lengths, fs, dio_options, time_axis, f0, f0_stride)
               : world_b200_dio_batch(h, x, m, x_stride, x_lengths, fs, &opt->dio, time_axis, f0, f0_stride);
  if (!rc) rc = world_b200_stonemask_batch(h, x, m, x_stride, x_lengths, fs, time_axis, f0, f0_lengths, f0_stride, f0);
  return rc;
}

}  // namespace wb

extern "C" {

int world_b200_frames(int fs, int x_length, double frame_period) {
  return frames_for(fs, x_length, frame_period);
}

int world_b200_create(int device, WorldB200 **out) {
  if (!out) return WORLD_B200_EINVAL;
  *out = nullptr;
  WorldB200 *h = new WorldB200;
  h->c.device = device;
#ifndef WB_EMU
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0 || device < 0 || device >= count) {
    fprintf(stderr, "world_b200: no usable CUDA device (%s); this library has no CPU path\n",
            e != cudaSuccess ? cudaGetErrorString(e) : "device index out of range");
    delete h;
    return WORLD_B200_ECUDA;
  }
  if (cudaSetDevice(device) != cudaSuccess) { delete h; return WORLD_B200_ECUDA; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->c.sm_count = prop.multiProcessorCount;
  // default scratch budget: a third of what is free now, between 4 and 64 GiB (an H100 has 80 GB; the
  // larger the passes, the fewer launches of the latency-bound per-utterance kernels)
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
    size_t want = free_b / 3;
    if (want > ((size_t)64 << 30)) want = (size_t)64 << 30;
    if (want < ((size_t)4 << 30)) want = (size_t)4 << 30;
    h->c.scratch_budget = want;
  }
#endif
  int rc = ctx_init_tables(&h->c);
  if (rc) {
    fprintf(stderr, "world_b200: context creation failed: %s\n", h->c.last_error.c_str());
    delete h;
    return rc;
  }
  *out = h;
  return 0;
}

void world_b200_destroy(WorldB200 *h) {
  if (!h) return;
  DeviceGuard guard_(&h->c);
  dev_sync(&h->c);
  for (int l = 0; l < 2; ++l) {
    if (h->lane[l]) world_b200_destroy(h->lane[l]);
#ifndef WB_EMU
    if (h->lane_stream[l]) cudaStreamDestroy((cudaStream_t)h->lane_stream[l]);
    if (h->ev_join[l]) cudaEventDestroy((cudaEvent_t)h->ev_join[l]);
#endif
  }
#ifndef WB_EMU
  if (h->ev_fork) cudaEventDestroy((cudaEvent_t)h->ev_fork);
  for (void *e : h->ev_slice) cudaEventDestroy((cudaEvent_t)e);
#endif
  if (h->comm) comm_destroy(h->comm);
  dev_free(h->c.twiddle);
  dev_free(h->c.twiddle_sized);
  dev_free(h->c.rng_jump);
  dev_free(h->c.status_dev);
  dev_free(h->c.arena.base);
  dev_free(h->lens_dev);
  for (auto &b : h->c.pool) dev_free(b.p);
#ifndef WB_EMU
  if (h->c.staging.base) {
    cudaFreeHost(h->c.staging.base);
    for (int i = 0; i < 2; ++i) cudaEventDestroy((cudaEvent_t)h->c.staging.left_event[i]);
  }
#endif
  delete h;
}

int world_b200_set_stream(WorldB200 *h, void *stream) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  if (h->c.stream != (wb_stream_t)stream) {
    // scratch arena and staging ring are reused in stream order: drain the old stream before switching
    int rc = dev_sync(&h->c);
    if (rc) return rc;
    h->c.stream = (wb_stream_t)stream;
  }
  return 0;
}

int world_b200_trim(WorldB200 *h) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  int rc = dev_sync(&h->c);
  for (int l = 0; l < 2; ++l)
    if (h->lane[l]) world_b200_trim(h->lane[l]);
  pool_trim(&h->c);
  dev_free(h->c.arena.base);
  h->c.arena = Arena();
  return rc;
}

int world_b200_set_scratch_budget(WorldB200 *h, unsigned long long bytes) {
  if (!h || bytes < ((unsigned long long)64 << 20)) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  h->c.scratch_budget = (size_t)bytes;
  return 0;
}

int world_b200_synchronize(WorldB200 *h) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  int rc = dev_sync(&h->c);
  if (rc) return rc;
  for (int l = 0; l < 2; ++l)
    if (h->lane[l]) {   // frames that hit an undefined case inside world_b200_analyze_batch set the lane's status word
      rc = world_b200_synchronize(h->lane[l]);
      if (rc) { h->c.last_error = h->lane[l]->c.last_error; return rc; }
    }
  int status = 0;
  rc = dev_memcpy_d2h(&h->c, &status, h->c.status_dev, sizeof(int));
  if (!rc) rc = dev_sync(&h->c);
  if (rc) return rc;
  if (status) {
    char msg[256];
    snprintf(msg, sizeof msg,
             "device status 0x%x: %s%s%s%s", status,
             (status & 1) ? "[analysis window longer than fft_size: f0 below the fft_size floor] " : "",
             (status & 2) ? "[smoothing width exceeds the spectrum] " : "",
             (status & 4) ? "[scratch overflow] " : "",
             (status & 8) ? "[randn stream past the 2^31 draws per utterance it reproduces] " : "");
    h->c.last_error = msg;
    dev_memset(&h->c, h->c.status_dev, 0, sizeof(int));
    return WORLD_B200_EDOMAIN;
  }
  return 0;
}

const char *world_b200_last_error(const WorldB200 *h) { return h ? h->c.last_error.c_str() : "null context"; }

unsigned long long world_b200_launch_count(const WorldB200 *) { return wb::g_launches; }

int world_b200_cheaptrick_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                                int f0_stride, const CheapTrickOption *opt, double *spectrogram) {
  if (!h || !x || !time_axis || !f0 || !opt || !spectrogram || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  int rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, f0_lengths, &b);
  if (rc) return rc;
  return cheaptrick_run(&h->c, b, opt->q1, opt->fft_size, spectrogram);
}

int world_b200_d4c_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                         const double *time_axis, const double *f0, const int *f0_lengths, int f0_stride,
                         int fft_size, const D4COption *opt, double *aperiodicity) {
  if (!h || !x || !time_axis || !f0 || !opt || !aperiodicity || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  int rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, f0_lengths, &b);
  if (rc) return rc;
  return d4c_run(&h->c, b, fft_size, opt->threshold, aperiodicity);
}

int world_b200_cheaptrick_coded_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                      int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                                      int f0_stride, const CheapTrickOption *opt, int number_of_dimensions,
                                      double *coded_spectral_envelope) {
  if (!h || !x || !time_axis || !f0 || !opt || !coded_spectral_envelope || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  CodecTables t;
  int rc = codec_sp_tables(&h->c, fs, opt->fft_size, number_of_dimensions, &t);
  if (rc) return rc;
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, f0_lengths, &b);
  if (rc) return rc;
  return cheaptrick_run(&h->c, b, opt->q1, opt->fft_size, nullptr, &t, coded_spectral_envelope);
}

int world_b200_d4c_coded_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                               const double *time_axis, const double *f0, const int *f0_lengths, int f0_stride,
                               int fft_size, const D4COption *opt, double *coded_aperiodicity) {
  if (!h || !x || !time_axis || !f0 || !opt || n < 0 || fs <= 0 || fft_size < 2) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  CodecTables t;
  int rc = codec_ap_tables(&h->c, fs, fft_size, &t);
  if (rc) return rc;
  if (t.dims == 0) return 0;        // nothing to write below 12 kHz, like the reference's empty loops
  if (!coded_aperiodicity) return WORLD_B200_EINVAL;
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, f0_lengths, &b);
  if (rc) return rc;
  return d4c_run(&h->c, b, fft_size, opt->threshold, nullptr, &t, coded_aperiodicity);
}

int world_b200_stonemask_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                               int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                               int f0_stride, double *refined_f0) {
  if (!h || !x || !time_axis || !f0 || !refined_f0 || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  int rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, f0_lengths, &b);
  if (rc) return rc;
  return stonemask_run(&h->c, b, refined_f0);
}

static int f0_lengths_from_x(int n, int x_stride, const int *x_lengths, int fs, double frame_period,
                             int f0_stride, std::vector<int> *out, std::string *err) {
  out->resize(n);
  for (int i = 0; i < n; ++i) {
    const int xl = x_lengths ? x_lengths[i] : x_stride;
    (*out)[i] = frames_for(fs, xl, frame_period);
    if ((*out)[i] > f0_stride) {
      *err = "f0_stride smaller than the frame count of an utterance";
      return WORLD_B200_EINVAL;
    }
  }
  return 0;
}

// opt: one option for every utterance, or (per_utt) an array of n
static int dio_batch_impl(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                          const DioOption *opt, bool per_utt, double *time_axis, double *f0, int f0_stride) {
  if (!h || !x || !time_axis || !f0 || !opt || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  if (per_utt && n > 0) {
    // every band list too, before the lengths are uploaded: a bad option queues nothing on the device
    const int rc = check_dio_options(&h->c, opt, n, opt[0].frame_period, opt[0].speed, fs);
    if (rc) return rc;
  }
  std::vector<int> fl;
  int rc = f0_lengths_from_x(n, x_stride, x_lengths, fs, opt->frame_period, f0_stride, &fl, &h->c.last_error);
  if (rc) return rc;
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, fl.data(), &b);
  if (rc) return rc;
  b.x_len_host = x_lengths;
  std::vector<DioParams> p(per_utt ? (n > 0 ? n : 1) : 1);
  for (size_t u = 0; u < p.size(); ++u)
    p[u] = {opt[u].f0_floor, opt[u].f0_ceil, opt[u].channels_in_octave, opt[u].frame_period, opt[u].allowed_range,
            opt[u].speed};
  return dio_run(&h->c, b, p.data(), per_utt, time_axis, f0);
}

int world_b200_dio_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                         const DioOption *opt, double *time_axis, double *f0, int f0_stride) {
  return dio_batch_impl(h, x, n, x_stride, x_lengths, fs, opt, false, time_axis, f0, f0_stride);
}

int world_b200_dio_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                 const DioOption *dio_options, double *time_axis, double *f0, int f0_stride) {
  return dio_batch_impl(h, x, n, x_stride, x_lengths, fs, dio_options, true, time_axis, f0, f0_stride);
}

// opt: one option for every utterance, or (per_utt) an array of n
static int harvest_batch_impl(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                              const HarvestOption *opt, bool per_utt, double *time_axis, double *f0, int f0_stride) {
  if (!h || !x || !time_axis || !f0 || !opt || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  if (per_utt && n > 0) {
    // every range too, before the lengths are uploaded: a bad option queues nothing on the device
    const int rc = check_harvest_options(&h->c, opt, n, opt[0].frame_period, fs);
    if (rc) return rc;
  }
  std::vector<int> fl;
  int rc = f0_lengths_from_x(n, x_stride, x_lengths, fs, opt->frame_period, f0_stride, &fl, &h->c.last_error);
  if (rc) return rc;
  Batch b;
  b.x = x; b.n = n; b.x_stride = x_stride; b.fs = fs; b.time_axis = time_axis; b.f0 = f0; b.f_stride = f0_stride;
  rc = upload_lengths(h, n, x_stride, x_lengths, f0_stride, fl.data(), &b);
  if (rc) return rc;
  std::vector<int> l1(n > 0 ? n : 1);
  for (int i = 0; i < n; ++i) l1[i] = frames_for(fs, x_lengths ? x_lengths[i] : x_stride, 1.0);
  b.l1_host = l1.data();
  b.x_len_host = x_lengths;
  std::vector<HarvestParams> p(per_utt ? (n > 0 ? n : 1) : 1);
  for (size_t u = 0; u < p.size(); ++u) p[u] = {opt[u].f0_floor, opt[u].f0_ceil, opt[u].frame_period};
  return harvest_run(&h->c, b, p.data(), per_utt, time_axis, f0);
}

int world_b200_harvest_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                             int fs, const HarvestOption *opt, double *time_axis, double *f0, int f0_stride) {
  return harvest_batch_impl(h, x, n, x_stride, x_lengths, fs, opt, false, time_axis, f0, f0_stride);
}

int world_b200_harvest_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                     const HarvestOption *harvest_options, double *time_axis, double *f0,
                                     int f0_stride) {
  return harvest_batch_impl(h, x, n, x_stride, x_lengths, fs, harvest_options, true, time_axis, f0, f0_stride);
}

// The whole chain on device arrays, cut into utterance slices that alternate between two lanes (sibling contexts
// on their own non-blocking streams).  Per slice the stages run in order on the lane's stream; the two lanes run
// concurrently, so the latency-bound per-utterance kernels of one slice (contour tracking, candidate clean-up, the
// draw stream, decimation) execute under the FP64-bound kernels of the other.  Ordered after the work already on the
// context's stream; that stream waits for both lanes before the function returns (no host synchronisation).
// gather = false: time_axis / f0 / spectrogram / aperiodicity hold this call's n utterances.
// gather = true (multi-GPU): they are the FULL arrays of n_ranks * n utterances; this rank computes into block `rank`
// and every finished slice is broadcast to the other ranks on the communication stream while the next one is computed.
// harvest_options / dio_options: nullptr, or one option per utterance of the chain's F0 method (at most one of the two;
// check_chain_f0_options); the slices split the array with the utterances.
// nbit: 0 = x holds doubles; 8/16/24/32 = little-endian PCM, converted slice by slice on the lane that analyses it.
// dims: 0 = spectrogram / aperiodicity receive the fft_size/2+1-bin rows; > 0 = they receive the coded rows
// (number_of_dimensions / GetNumberOfAperiodicities(fs) values per frame) straight from the fused frame kernels.
static int analyze_batch_impl(WorldB200 *h, const void *x, int nbit, int n, int x_stride, const int *x_lengths, int fs,
                              const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                              const DioOption *dio_options, int dims, double *time_axis, double *f0, int f0_stride,
                              double *spectrogram, double *aperiodicity, bool gather) {
  if (!h || !x || !opt || !time_axis || !f0 || n < 0 || fs <= 0 || x_stride <= 0 || f0_stride <= 0) return WORLD_B200_EINVAL;
  if ((spectrogram || aperiodicity) && opt->cheaptrick.fft_size < 16) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  const char *who = dims ? "analyze_coded_batch" : "analyze_batch";
  if (nbit != 0 && nbit != 8 && nbit != 16 && nbit != 24 && nbit != 32) {
    h->c.last_error = std::string(who) + ": nbit must be 0, 8, 16, 24 or 32";
    return WORLD_B200_EINVAL;
  }
  {
    const int rc = check_chain_f0_options(&h->c, opt, harvest_options, dio_options, n, fs, who);
    if (rc) return rc;
  }
  const int bins = opt->cheaptrick.fft_size / 2 + 1;
  const int n_ap = dims ? GetNumberOfAperiodicities(fs) : 0;
  if (dims) {
    // the codec tables of every slice, built once here so that a bad dimension count or fft_size queues nothing
    CodecTables t;
    int rc = spectrogram ? codec_sp_tables(&h->c, fs, opt->cheaptrick.fft_size, dims, &t) : 0;
    if (!rc && aperiodicity) rc = codec_ap_tables(&h->c, fs, opt->cheaptrick.fft_size, &t);
    if (rc) return rc;
    if (n_ap == 0) aperiodicity = nullptr;   // no bands below 12 kHz: nothing to write, D4C is skipped
  }
  const size_t sp_row = dims ? (size_t)dims : (size_t)bins, ap_row = dims ? (size_t)n_ap : (size_t)bins;
  if (n == 0) return 0;
  const double frame_period = opt->f0_method == WORLD_B200_F0_HARVEST ? opt->harvest.frame_period : opt->dio.frame_period;
  // every utterance's length and frame count up front: a bad one queues no slice
  std::vector<int> fl(n);
  for (int i = 0; i < n; ++i) {
    const int xl = x_lengths ? x_lengths[i] : x_stride;
    if (xl < 1 || xl > x_stride) { h->c.last_error = "utterance length outside its padded row"; return WORLD_B200_EINVAL; }
    fl[i] = frames_for(fs, xl, frame_period);
    if (fl[i] > f0_stride) { h->c.last_error = "f0_stride smaller than the frame count of an utterance"; return WORLD_B200_EINVAL; }
  }
  size_t my_block = 0;
  if (gather) {
    if (!h->comm) { h->c.last_error = std::string(who) + "_allgather: no communicator (world_b200_comm_init)"; return WORLD_B200_EINVAL; }
    my_block = (size_t)comm_rank(h->comm) * (size_t)n;
    time_axis += my_block * f0_stride; f0 += my_block * f0_stride;
    if (spectrogram) spectrogram += my_block * f0_stride * sp_row;
    if (aperiodicity) aperiodicity += my_block * f0_stride * ap_row;
  }
  // two slices (one per lane) overlap best on one GPU (more slices only add launches); with the
  // gather the exposed tail is the LAST slice's transfer, so more, smaller slices win there
  int n_slices = gather ? 10 : 2;
  if (const char *e = getenv("WB_LANE_SLICES")) n_slices = atoi(e);
  n_slices = imax(1, imin(n_slices, n));
  // Slice boundaries.  From six slices on the slices taper (weights 3 .. 3 2 2 1 1): the two lanes finish together, so
  // the transfers of the LAST slice of each lane are the exposed tail of the gather -- they should be small, while
  // small slices everywhere would only multiply the launches of the latency-bound kernels.
  std::vector<int> bounds(n_slices + 1, 0);
  {
    std::vector<int> wgt(n_slices, 1);
    if (n_slices >= 6)
      for (int s = 0; s < n_slices; ++s) wgt[s] = s >= n_slices - 2 ? 1 : (s >= n_slices - 4 ? 2 : 3);
    long long total = 0, run = 0;
    for (int s = 0; s < n_slices; ++s) total += wgt[s];
    for (int s = 0; s < n_slices; ++s) { run += wgt[s]; bounds[s + 1] = (int)((long long)n * run / total); }
  }
  WorldB200 *lanes[2] = {h, h};
#ifndef WB_EMU
  if (n_slices > 1) {
    for (int l = 0; l < 2; ++l) {
      if (!h->lane[l]) {
        int rc = world_b200_create(h->c.device, &h->lane[l]);
        if (rc) { h->c.last_error = "analyze_batch: cannot create a lane context"; return rc; }
        cudaStream_t st;
        cudaEvent_t ev;
        // equal (lowest) priority for both lanes: giving one lane the highest priority was measured slower;
        // only the communication stream outranks them (wb_multi.cu)
        if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
          h->c.last_error = "analyze_batch: cannot create a lane stream";
          return WORLD_B200_ECUDA;
        }
        h->lane_stream[l] = st; h->ev_join[l] = ev;
        h->lane[l]->c.stream = st;
      }
      h->lane[l]->c.scratch_budget = h->c.scratch_budget / 2;
      lanes[l] = h->lane[l];
    }
    if (!h->ev_fork) {
      cudaEvent_t ev;
      if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return WORLD_B200_ECUDA;
      h->ev_fork = ev;
    }
    cudaEventRecord((cudaEvent_t)h->ev_fork, h->c.stream);
    for (int l = 0; l < 2; ++l) cudaStreamWaitEvent((cudaStream_t)h->lane_stream[l], (cudaEvent_t)h->ev_fork, 0);
  }
#endif
  int rc = 0;
  // nbit != 0: each lane converts its slice into a float64 buffer, which the slice's three stages then read.  A lane
  // runs its slices in stream order, so one buffer per lane, sized for its largest slice, serves all of them.  It comes
  // from the lane's pool, not its arena (the stage drivers reset the arena when they return), and its bytes come out
  // of the lane's scratch budget; the stages keep at least half of that budget (less would only mean more passes).
  double *xbuf[2] = {nullptr, nullptr};
  const size_t own_budget = h->c.scratch_budget;   // restored on return when the context is its own (only) lane
  if (nbit) {
    const bool one_lane = lanes[0] == lanes[1];
    int most[2] = {0, 0};
    for (int s = 0; s < n_slices; ++s) {
      const int l = one_lane ? 0 : (s & 1);
      most[l] = imax(most[l], bounds[s + 1] - bounds[s]);
    }
    for (int l = 0; l < 2 && !rc; ++l) {
      if (most[l] == 0) continue;
      Ctx *c = &lanes[l]->c;
      const size_t bytes = (size_t)most[l] * x_stride * sizeof(double);
      xbuf[l] = (double *)pool_acquire(c, bytes);
      if (!xbuf[l]) { h->c.last_error = c->last_error; rc = WORLD_B200_ENOMEM; }
      c->scratch_budget -= bytes < c->scratch_budget / 2 ? bytes : c->scratch_budget / 2;
    }
    if (one_lane) xbuf[1] = xbuf[0];
  }
#ifndef WB_EMU
  // multi-GPU: the full arrays and how a finished slice reaches the other ranks -- pushed into their (IPC-mapped)
  // arrays by the copy engines where that is possible, grouped NCCL broadcasts otherwise (wb_multi.cu).  An array
  // that is not computed is NULL here, so it is neither exported nor sent.
  double *fulls[4] = {time_axis - my_block * f0_stride, f0 - my_block * f0_stride,
                      spectrogram ? spectrogram - my_block * f0_stride * sp_row : nullptr,
                      aperiodicity ? aperiodicity - my_block * f0_stride * ap_row : nullptr};
  const size_t full_elems[4] = {(size_t)f0_stride, (size_t)f0_stride, spectrogram ? (size_t)f0_stride * sp_row : 0,
                                aperiodicity ? (size_t)f0_stride * ap_row : 0};
  const bool exchange = gather && comm_ranks(h->comm) > 1;
  bool push = false;
  if (!rc && exchange && !getenv("WB_NO_P2P")) {
    std::string err;
    const int pr = comm_p2p_prepare(h->comm, 4, fulls, &err);
    if (pr == 2) { h->c.last_error = err; rc = WORLD_B200_ECUDA; }
    push = pr == 0;
  }
#endif
  for (int s = 0; s < n_slices && !rc; ++s) {
    const int u0 = bounds[s], u1 = bounds[s + 1];
    const int m = u1 - u0;
    if (m <= 0) continue;
    WorldB200 *L = lanes[s & 1];
    const int *xl = x_lengths ? x_lengths + u0 : nullptr;
    const double *xs = xbuf[s & 1];
    if (nbit)
      rc = world_b200_pcm_to_double_batch(L, (const unsigned char *)x + (size_t)u0 * x_stride * (nbit / 8), nbit, m,
                                          x_stride, xl, xbuf[s & 1]);
    else
      xs = (const double *)x + (size_t)u0 * x_stride;
    double *ts = time_axis + (size_t)u0 * f0_stride, *fs_ = f0 + (size_t)u0 * f0_stride;
    const int *fls = fl.data() + u0;
    if (!rc)
      rc = run_f0_stage(L, xs, m, x_stride, xl, fs, opt, harvest_options ? harvest_options + u0 : nullptr,
                        dio_options ? dio_options + u0 : nullptr, fls, ts, fs_, f0_stride);
    double *sps = spectrogram ? spectrogram + (size_t)u0 * f0_stride * sp_row : nullptr;
    double *aps = aperiodicity ? aperiodicity + (size_t)u0 * f0_stride * ap_row : nullptr;
    if (!rc && sps)
      rc = dims ? world_b200_cheaptrick_coded_batch(L, xs, m, x_stride, xl, fs, ts, fs_, fls, f0_stride, &opt->cheaptrick,
                                                    dims, sps)
                : world_b200_cheaptrick_batch(L, xs, m, x_stride, xl, fs, ts, fs_, fls, f0_stride, &opt->cheaptrick, sps);
    if (!rc && aps)
      rc = dims ? world_b200_d4c_coded_batch(L, xs, m, x_stride, xl, fs, ts, fs_, fls, f0_stride,
                                             opt->cheaptrick.fft_size, &opt->d4c, aps)
                : world_b200_d4c_batch(L, xs, m, x_stride, xl, fs, ts, fs_, fls, f0_stride, opt->cheaptrick.fft_size,
                                       &opt->d4c, aps);
    if (rc && L != h) h->c.last_error = L->c.last_error;
#ifndef WB_EMU
    if (!rc && exchange) {
      // rows u0..u1 of every rank's block, as soon as this rank's are final (event on the lane's stream)
      while ((int)h->ev_slice.size() <= s) {
        cudaEvent_t ev;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return WORLD_B200_ECUDA;
        h->ev_slice.push_back(ev);
      }
      cudaEvent_t ev = (cudaEvent_t)h->ev_slice[s];
      cudaEventRecord(ev, L->c.stream);
      std::string err;
      const int g = push ? comm_p2p_push(h->comm, 4, full_elems, (size_t)n, (size_t)u0, (size_t)m, ev, &err)
                         : comm_gather_rows_multi(h->comm, 4, fulls, full_elems, (size_t)n, (size_t)u0, (size_t)m, ev, &err);
      if (g) { h->c.last_error = err; rc = WORLD_B200_ECUDA; }
    }
#endif
  }
#ifndef WB_EMU
  if (exchange) {
    std::string err;
    const int g = push ? comm_p2p_finish(h->comm, h->c.stream, &err) : comm_join(h->comm, h->c.stream, &err);
    if (g && !rc) { h->c.last_error = err; rc = WORLD_B200_ECUDA; }
  }
  if (lanes[0] != h)
    for (int l = 0; l < 2; ++l) {   // join even after an error: the caller's stream must not run ahead of the lanes
      cudaEventRecord((cudaEvent_t)h->ev_join[l], (cudaStream_t)h->lane_stream[l]);
      cudaStreamWaitEvent(h->c.stream, (cudaEvent_t)h->ev_join[l], 0);
    }
#endif
  // back to the pool while the lanes may still read them: a pooled buffer is only handed out again to work that is
  // ordered after this call's (the lane's next slices, or the host pipelines, whose uploads wait for the stream)
  pool_release(&lanes[0]->c, xbuf[0]);
  if (xbuf[1] != xbuf[0]) pool_release(&lanes[1]->c, xbuf[1]);
  h->c.scratch_budget = own_budget;
  return rc;
}

int world_b200_analyze_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                             const WorldB200AnalysisOption *opt, double *time_axis, double *f0, int f0_stride,
                             double *spectrogram, double *aperiodicity) {
  return analyze_batch_impl(h, x, 0, n, x_stride, x_lengths, fs, opt, nullptr, nullptr, 0, time_axis, f0, f0_stride,
                            spectrogram, aperiodicity, false);
}

int world_b200_analyze_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                     const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                     double *time_axis, double *f0, int f0_stride, double *spectrogram,
                                     double *aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  return analyze_batch_impl(h, x, 0, n, x_stride, x_lengths, fs, opt, harvest_options, nullptr, 0, time_axis, f0, f0_stride,
                            spectrogram, aperiodicity, false);
}

int world_b200_analyze_batch_dio_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                         int fs, const WorldB200AnalysisOption *opt, const DioOption *dio_options,
                                         double *time_axis, double *f0, int f0_stride, double *spectrogram,
                                         double *aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  return analyze_batch_impl(h, x, 0, n, x_stride, x_lengths, fs, opt, nullptr, dio_options, 0, time_axis, f0, f0_stride,
                            spectrogram, aperiodicity, false);
}

// ---- multi-GPU (SURVEY.md 8e): utterances sharded over ranks, outputs reassembled on every rank by NCCL
int world_b200_comm_unique_id(unsigned char *id, int id_bytes) {
  if (!id || id_bytes < 128) return WORLD_B200_EINVAL;
  std::string err;
  if (comm_unique_id(id, &err)) { fprintf(stderr, "world_b200: %s\n", err.c_str()); return WORLD_B200_ECUDA; }
  return 0;
}

int world_b200_comm_init(WorldB200 *h, int n_ranks, int rank, const unsigned char *id, int id_bytes) {
  if (!h || !id || id_bytes < 128 || n_ranks < 1 || rank < 0 || rank >= n_ranks) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  if (h->comm) { comm_destroy(h->comm); h->comm = nullptr; }
  std::string err;
  if (comm_create(n_ranks, rank, id, &h->comm, &err)) { h->c.last_error = err; return WORLD_B200_ECUDA; }
  return 0;
}

int world_b200_comm_destroy(WorldB200 *h) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  if (h->comm) { comm_destroy(h->comm); h->comm = nullptr; }
  return 0;
}

// In-place all-gather of an array of n_ranks blocks of rows_per_rank rows (row_elems doubles each): this rank's block
// is already in place.  Ordered after the work on the context's stream; that stream waits for the result.
int world_b200_allgather_rows(WorldB200 *h, double *full, unsigned long long row_elems, unsigned long long rows_per_rank) {
  if (!h || !full) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  if (!h->comm) { h->c.last_error = "allgather_rows: no communicator (world_b200_comm_init)"; return WORLD_B200_EINVAL; }
#ifndef WB_EMU
  if (comm_ranks(h->comm) > 1) {
    if (!h->ev_fork) {
      cudaEvent_t ev;
      if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return WORLD_B200_ECUDA;
      h->ev_fork = ev;
    }
    cudaEventRecord((cudaEvent_t)h->ev_fork, h->c.stream);
    std::string err;
    int g = comm_gather_rows(h->comm, full, (size_t)row_elems, (size_t)rows_per_rank, 0, (size_t)rows_per_rank,
                             (cudaEvent_t)h->ev_fork, &err);
    if (!g) g = comm_join(h->comm, h->c.stream, &err);
    if (g) { h->c.last_error = err; return WORLD_B200_ECUDA; }
  }
#endif
  return 0;
}

int world_b200_analyze_batch_allgather(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                       const WorldB200AnalysisOption *opt, double *time_axis_full, double *f0_full,
                                       int f0_stride, double *spectrogram_full, double *aperiodicity_full) {
  return analyze_batch_impl(h, x, 0, n, x_stride, x_lengths, fs, opt, nullptr, nullptr, 0, time_axis_full, f0_full, f0_stride,
                            spectrogram_full, aperiodicity_full, true);
}

int world_b200_analyze_batch_allgather_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                               int fs, const WorldB200AnalysisOption *opt,
                                               const HarvestOption *harvest_options, double *time_axis_full,
                                               double *f0_full, int f0_stride, double *spectrogram_full,
                                               double *aperiodicity_full) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  return analyze_batch_impl(h, x, 0, n, x_stride, x_lengths, fs, opt, harvest_options, nullptr, 0, time_axis_full, f0_full,
                            f0_stride, spectrogram_full, aperiodicity_full, true);
}

int world_b200_analyze_batch_allgather_dio_options(WorldB200 *h, const double *x, int n, int x_stride,
                                                   const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                   const DioOption *dio_options, double *time_axis_full,
                                                   double *f0_full, int f0_stride, double *spectrogram_full,
                                                   double *aperiodicity_full) {
  if (!dio_options) return WORLD_B200_EINVAL;
  return analyze_batch_impl(h, x, 0, n, x_stride, x_lengths, fs, opt, nullptr, dio_options, 0, time_axis_full, f0_full,
                            f0_stride, spectrogram_full, aperiodicity_full, true);
}

// The device chain with coded rows out (and PCM or doubles in): the checks of analyze_coded_host, then the slices of
// analyze_batch_impl with the fused coded frame kernels.
static int analyze_coded_batch_impl(WorldB200 *h, const void *x, int nbit, int n, int x_stride, const int *x_lengths,
                                    int fs, const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                    const DioOption *dio_options, int number_of_dimensions, double *time_axis,
                                    double *f0, int f0_stride, double *coded_spectral_envelope,
                                    double *coded_aperiodicity, bool gather) {
  if (!h || !opt) return WORLD_B200_EINVAL;
  if (number_of_dimensions < 1 || number_of_dimensions > opt->cheaptrick.fft_size / 4 + 1) {
    h->c.last_error = "analyze_coded_batch: number_of_dimensions must be in [1, fft_size/4 + 1]";
    return WORLD_B200_EINVAL;
  }
  return analyze_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, harvest_options, dio_options,
                            number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope, coded_aperiodicity,
                            gather);
}

int world_b200_analyze_coded_batch(WorldB200 *h, const void *x, int nbit, int n, int x_stride, const int *x_lengths,
                                   int fs, const WorldB200AnalysisOption *opt, int number_of_dimensions,
                                   double *time_axis, double *f0, int f0_stride, double *coded_spectral_envelope,
                                   double *coded_aperiodicity) {
  return analyze_coded_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, nullptr, nullptr, number_of_dimensions,
                                  time_axis, f0, f0_stride, coded_spectral_envelope, coded_aperiodicity, false);
}

int world_b200_analyze_coded_batch_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                           const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                           const HarvestOption *harvest_options, int number_of_dimensions,
                                           double *time_axis, double *f0, int f0_stride,
                                           double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  return analyze_coded_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, harvest_options, nullptr,
                                  number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope,
                                  coded_aperiodicity, false);
}

int world_b200_analyze_coded_batch_dio_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                               const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                               const DioOption *dio_options, int number_of_dimensions,
                                               double *time_axis, double *f0, int f0_stride,
                                               double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  return analyze_coded_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, nullptr, dio_options,
                                  number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope,
                                  coded_aperiodicity, false);
}

int world_b200_analyze_coded_batch_allgather(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                             const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                             int number_of_dimensions, double *time_axis_full, double *f0_full,
                                             int f0_stride, double *coded_spectral_envelope_full,
                                             double *coded_aperiodicity_full) {
  return analyze_coded_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, nullptr, nullptr, number_of_dimensions,
                                  time_axis_full, f0_full, f0_stride, coded_spectral_envelope_full,
                                  coded_aperiodicity_full, true);
}

int world_b200_analyze_coded_batch_allgather_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                                     const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                     const HarvestOption *harvest_options, int number_of_dimensions,
                                                     double *time_axis_full, double *f0_full, int f0_stride,
                                                     double *coded_spectral_envelope_full,
                                                     double *coded_aperiodicity_full) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  return analyze_coded_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, harvest_options, nullptr,
                                  number_of_dimensions, time_axis_full, f0_full, f0_stride,
                                  coded_spectral_envelope_full, coded_aperiodicity_full, true);
}

int world_b200_analyze_coded_batch_allgather_dio_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                                         const int *x_lengths, int fs,
                                                         const WorldB200AnalysisOption *opt,
                                                         const DioOption *dio_options, int number_of_dimensions,
                                                         double *time_axis_full, double *f0_full, int f0_stride,
                                                         double *coded_spectral_envelope_full,
                                                         double *coded_aperiodicity_full) {
  if (!dio_options) return WORLD_B200_EINVAL;
  return analyze_coded_batch_impl(h, x, nbit, n, x_stride, x_lengths, fs, opt, nullptr, dio_options,
                                  number_of_dimensions, time_axis_full, f0_full, f0_stride,
                                  coded_spectral_envelope_full, coded_aperiodicity_full, true);
}

// Per-kernel timing: enable, run, then fetch a JSON object {"kernel": {"launches": n, "ms": t}, ...}
// (CUDA events recorded on the context's stream around every launch; report() synchronises).
int world_b200_profile(WorldB200 *h, int enable) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  wb::g_prof_on = enable ? 1 : 0;
  return 0;
}

int world_b200_profile_report(WorldB200 *h, char *buf, unsigned long long cap) {
  if (!h || !buf || cap < 3) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  std::string out = "{";
#ifndef WB_EMU
  int rc = dev_sync(&h->c);
  if (rc) return rc;
  std::vector<std::string> names; std::vector<double> ms; std::vector<long> cnt;
  for (auto &r : g_prof) {
    float t = 0.f;
    cudaEventElapsedTime(&t, r.a, r.b);
    size_t k = 0;
    for (; k < names.size(); ++k) if (names[k] == r.name) break;
    if (k == names.size()) { names.push_back(r.name); ms.push_back(0.0); cnt.push_back(0); }
    ms[k] += t; cnt[k] += 1;
    g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
  }
  g_prof.clear();
  for (size_t k = 0; k < names.size(); ++k) {
    char item[256];
    snprintf(item, sizeof item, "%s\"%s\": {\"launches\": %ld, \"ms\": %.6f}", k ? ", " : "", names[k].c_str(), cnt[k], ms[k]);
    out += item;
  }
#endif
  out += "}";
  if (out.size() + 1 > cap) return WORLD_B200_EINVAL;
  memcpy(buf, out.c_str(), out.size() + 1);
  return 0;
}

// FP64 FMA peak of this device (the roofline the path is actually bound by; MEASURED_PEAKS.json
// has no FP64 figure): 8 independent DFMA chains per thread, timed with CUDA events.
#ifndef WB_EMU
__global__ void fp64_peak_kernel(double *out, int iters) {
  double a0 = threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  const double m = 1.0000000001, c = 0.5;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}
#endif

int world_b200_fp64_peak(WorldB200 *h, double *tflops) {
  if (!h || !tflops) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  *tflops = 0.0;
#ifndef WB_EMU
  Ctx *ctx = &h->c;
  const int blocks = ctx->sm_count * 8, threads = 256, iters = 1 << 15;
  unsigned char *blk = arena_block(ctx, (size_t)blocks * threads * 8);
  if (!blk) return WORLD_B200_ENOMEM;
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {
    cudaEventRecord(a, ctx->stream);
    fp64_peak_kernel<<<blocks, threads, 0, ctx->stream>>>((double *)blk, iters);
    cudaEventRecord(b, ctx->stream);
    cudaEventSynchronize(b);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, a, b);
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(a); cudaEventDestroy(b);
  *tflops = (double)blocks * threads * iters * 8 * 2 / (best * 1e-3) / 1e12;
  return dev_check(ctx, "fp64_peak");
#else
  return 0;
#endif
}

// FP64 tensor-core (DMMA) peak: the same harness with 8 independent mma.m16n8k4.f64 chains per warp
// (16 x 8 x 4 MACs per instruction) instead of DFMA chains.
#ifndef WB_EMU
__global__ void fp64_tensor_peak_kernel(double *out, int iters) {
  double c[8][4];
  const double a = 1e-3 * (threadIdx.x & 7), b = 1e-3;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    for (int r = 0; r < 4; ++r) c[k][r] = k + r;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                   : "+d"(c[k][0]), "+d"(c[k][1]), "+d"(c[k][2]), "+d"(c[k][3]) : "d"(a), "d"(a), "d"(b));
  }
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) s += c[k][0] + c[k][1] + c[k][2] + c[k][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
#endif

int world_b200_fp64_tensor_peak(WorldB200 *h, double *tflops) {
  if (!h || !tflops) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  *tflops = 0.0;
#ifndef WB_EMU
  Ctx *ctx = &h->c;
  const int blocks = ctx->sm_count * 8, threads = 256, iters = 1 << 12;
  unsigned char *blk = arena_block(ctx, (size_t)blocks * threads * 8);
  if (!blk) return WORLD_B200_ENOMEM;
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {
    cudaEventRecord(a, ctx->stream);
    fp64_tensor_peak_kernel<<<blocks, threads, 0, ctx->stream>>>((double *)blk, iters);
    cudaEventRecord(b, ctx->stream);
    cudaEventSynchronize(b);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, a, b);
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(a); cudaEventDestroy(b);
  // per warp and iteration: 8 MMAs of 16 x 8 x 4 multiply-adds
  *tflops = (double)blocks * (threads / 32) * iters * 8 * (16 * 8 * 4) * 2 / (best * 1e-3) / 1e12;
  return dev_check(ctx, "fp64_tensor_peak");
#else
  return 0;
#endif
}

// Known-answer hook for the shared-memory FFT: r2c of n = 2^lg reals (n/2+1 complex out), one CTA.
namespace wb {
WB_KERNEL(128, 1) rfft_test_kernel(const double *x, int n, int lg, double *out, const double2 *tw) {
  WB_DYN_SMEM(double, buf);
  for (int i = WB_TID; i < n + 2; i += WB_NTH) buf[i] = i < n ? x[i] : 0.0;
  WB_SYNC();
  rfft_forward(buf, lg, tw);
  for (int i = WB_TID; i < n + 2; i += WB_NTH) out[i] = buf[i];
}
// the Stockham path of the frame kernels (wb_fft.cuh, round 2): packed padded input, ping-pong, fused unpack
WB_KERNEL(128, 1) sfft_test_kernel(const double *x, int n, int lg, double *out, const double2 *tw) {
  WB_DYN_SMEM(double, buf);
  const int slots = WB_FPAD_SLOTS(n >> 1);
  double2 *a = reinterpret_cast<double2 *>(buf), *b = a + slots;
  for (int i = WB_TID; i < n; i += WB_NTH) buf[rpad(i)] = x[i];
  WB_SYNC();
  const double2 *z = sfft_forward(a, b, lg - 1, tw);
  rfft_unpack(z, lg, tw, [&](int k, double2 v) { out[2 * k] = v.x; out[2 * k + 1] = v.y; });
}
}  // namespace wb

int world_b200_sfft_test(WorldB200 *h, const double *x_dev, int n, double *out_dev) {
  if (!h || !x_dev || !out_dev) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  int lg = 0;
  while ((1 << lg) < n) ++lg;
  if ((1 << lg) != n || n < 4 || n > WB_TW_N) return WORLD_B200_EINVAL;
  Ctx *ctx = &h->c;
  const size_t smem = (size_t)2 * WB_FPAD_SLOTS(n >> 1) * 16;
#ifndef WB_EMU
  cudaFuncSetAttribute(sfft_test_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  WB_LAUNCH_COOP(sfft_test_kernel, dim3(1), 128, smem, ctx->stream, x_dev, n, lg, out_dev, ctx->twiddle);
  return dev_check(ctx, "sfft_test");
}

int world_b200_rfft_test(WorldB200 *h, const double *x_dev, int n, double *out_dev) {
  if (!h || !x_dev || !out_dev) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  int lg = 0;
  while ((1 << lg) < n) ++lg;
  if ((1 << lg) != n || n < 4 || n > WB_TW_N) return WORLD_B200_EINVAL;
  Ctx *ctx = &h->c;
  const size_t smem = (size_t)(n + 2) * 8;
#ifndef WB_EMU
  cudaFuncSetAttribute(rfft_test_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  WB_LAUNCH_COOP(rfft_test_kernel, dim3(1), 128, smem, ctx->stream, x_dev, n, lg, out_dev, ctx->twiddle);
  return dev_check(ctx, "rfft_test");
}

// Known-answer hook: the first n_draws randn() draws after randn_reseed(), as the raw 32-bit
// sums (value = sum / 2^28 - 6), written to a device buffer of n_draws uint32.
int world_b200_randn_stream(WorldB200 *h, unsigned n_draws, unsigned *out_dev) {
  return world_b200_randn_window(h, 0, n_draws, out_dev);
}

// Known-answer hook: draws [first, first + n) of the same stream, through the kernel the stages use.
int world_b200_randn_window(WorldB200 *h, unsigned long long first, unsigned n, unsigned *out_dev) {
  if (!h || !out_dev) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  if (first > WB_RNG_REACH || n > WB_RNG_REACH - first) {
    ctx->last_error = "randn_window: the stream is reproduced up to draw 2^31";
    return WORLD_B200_EINVAL;
  }
  if (n == 0) return 0;
  unsigned char *blk = arena_block(ctx, 256);
  if (!blk) return WORLD_B200_ENOMEM;
  const unsigned end = (unsigned)(first + n);
  int rc = dev_memcpy_h2d(ctx, blk, &end, sizeof(unsigned));
  if (rc) return rc;
  rng_fill(ctx, reinterpret_cast<unsigned *>(blk), out_dev, 0, end, 1, (unsigned)first);
  return dev_check(ctx, "randn_window");
}

// ---- option helpers: pure host arithmetic, the reference's expressions verbatim in meaning
void InitializeDioOption(DioOption *o) {
  o->channels_in_octave = 2.0; o->f0_ceil = 800.0; o->f0_floor = 71.0; o->frame_period = 5;
  o->speed = 1; o->allowed_range = 0.1;
}
void InitializeHarvestOption(HarvestOption *o) { o->f0_ceil = 800.0; o->f0_floor = 71.0; o->frame_period = 5; }
void InitializeD4COption(D4COption *o) { o->threshold = 0.85; }
int GetFFTSizeForCheapTrick(int fs, const CheapTrickOption *o) {
  return static_cast<int>(pow(2.0, 1.0 + static_cast<int>(log(3.0 * fs / o->f0_floor + 1) / wb::kLog2)));
}
double GetF0FloorForCheapTrick(int fs, int fft_size) { return 3.0 * fs / (fft_size - 3.0); }
void InitializeCheapTrickOption(int fs, CheapTrickOption *o) {
  o->q1 = -0.15; o->f0_floor = 71.0; o->fft_size = GetFFTSizeForCheapTrick(fs, o);
}
int GetSamplesForDIO(int fs, int x_length, double frame_period) { return frames_for(fs, x_length, frame_period); }
int GetSamplesForHarvest(int fs, int x_length, double frame_period) { return frames_for(fs, x_length, frame_period); }

void world_b200_default_analysis_option(int fs, int f0_method, WorldB200AnalysisOption *o) {
  o->f0_method = f0_method;
  InitializeDioOption(&o->dio);
  InitializeHarvestOption(&o->harvest);
  InitializeCheapTrickOption(fs, &o->cheaptrick);
  InitializeD4COption(&o->d4c);
}

}  // extern "C"
