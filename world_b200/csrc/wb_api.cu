// wb_api.cu -- context, scratch arena and the extern "C" ABI declared in include/world_b200.h,
// plus the legacy single-utterance entry points of include/world/*.h implemented as n_utts = 1
// batches (reference boundary: src/world/{dio,harvest,stonemask,cheaptrick,d4c}.h).
#include "wb_chain.h"
#include "wb_f0common.cuh"
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <vector>
#include <string>
#include <algorithm>
#include <climits>
#include <cmath>
#include <type_traits>

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
// WB_ARENA_POISON=<byte> (test hook, README): the block is filled with that byte (stream ordered) before it is
// returned, so a stage that reads scratch it did not write this call sees the poison instead of earlier values.  A
// value that is not one byte (0..255, decimal or 0x hex) fails the call rather than poisoning with something else.
unsigned char *arena_block(Ctx *ctx, size_t bytes) {
  Arena &a = ctx->arena;
  int poison = -1;
  if (const char *e = getenv("WB_ARENA_POISON")) {
    char *end = nullptr;
    const long v = strtol(e, &end, 0);
    if (end == e || *end != '\0' || v < 0 || v > 255) {
      ctx->last_error = std::string("WB_ARENA_POISON=\"") + e + "\": not a byte value (0..255, decimal or 0x hex)";
      return nullptr;
    }
    poison = (int)v;
  }
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
  if (poison >= 0 && dev_memset(ctx, a.base, poison, bytes)) return nullptr;
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
  if (!rc && !rng_table_reserve(ctx, 1)) rc = WORLD_B200_ENOMEM;
  if (!rc) rc = dev_sync(ctx);
  return rc;
}

}  // namespace wb

using namespace wb;

// ------------------------------------------------------------------------------------------
// The Batch of n utterances' rows, with their lengths x_len / f_len [n] (checked by the caller) uploaded.  offs (packed
// inputs): the host offsets x_off [n] and f_off [n + 1], uploaded after the lengths for b->x_off / b->f_off.
static int load_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_len, int fs,
                      const double *time_axis, const double *f0, const int *f_len, int f_stride, Batch *b,
                      const std::vector<long long> *offs = nullptr) {
  Ctx *ctx = &h->c;
  b->x = x; b->n = n; b->x_stride = x_stride; b->fs = fs; b->time_axis = time_axis; b->f0 = f0; b->f_stride = f_stride;
  // the offsets follow the 2n lengths, at an 8-byte boundary
  const size_t ints = (size_t)2 * n + (offs ? 2 * offs->size() : 0);
  if (ints > h->lens_cap) {
    dev_sync(ctx);
    dev_free(h->lens_dev);
    h->lens_cap = ints + 64;
    h->lens_dev = (int *)dev_malloc(ctx, h->lens_cap * sizeof(int));
    if (!h->lens_dev) { h->lens_cap = 0; return WORLD_B200_ENOMEM; }
  }
  std::vector<int> tmp(ints);
  if (offs) {
    memcpy(tmp.data() + 2 * n, offs->data(), offs->size() * 8);
    b->x_off = (const long long *)(h->lens_dev + 2 * n);
    b->f_off = b->x_off + n;
  }
  int mx = 0, mf = 0;
  for (int i = 0; i < n; ++i) {
    tmp[i] = x_len[i]; tmp[n + i] = f_len[i];
    mx = imax(mx, x_len[i]);
    mf = imax(mf, f_len[i]);
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
  dev_free(h->c.rng_table);
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
  dev_free(h->c.rng_table);
  h->c.rng_table = nullptr;
  h->c.rng_table_len = 0;
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

}  // extern "C"

namespace wb {
std::string packed_lengths(const char *name, const char *unit, int n, const long long *off, int least,
                           std::vector<int> *len) {
  if (!off) return std::string(name) + " must be given";
  if (off[0] != 0) return std::string(name) + "[0] = " + std::to_string(off[0]) + " is not 0";
  len->resize(n);
  for (int u = 0; u < n; ++u) {
    const long long l = off[u + 1] - off[u];
    if (l < least || l > INT_MAX)
      return std::string(name) + " must increase by " + std::to_string(least) + " to INT_MAX " + unit +
             " per utterance, not " + std::to_string(l) + " (utterance " + std::to_string(u) + ")";
    (*len)[u] = (int)l;
  }
  return "";
}
}  // namespace wb

// The packed layout's offsets: x_offsets[0] == 0 and every utterance 1 .. INT_MAX samples long.  Fills x_len [n] and
// f_off [n + 1] (frames at frame_period ms); "" when the offsets are good, else the first broken rule.
static std::string packed_layout(int fs, int n, const long long *x_offsets, double frame_period, std::vector<int> *x_len,
                                 std::vector<long long> *f_off) {
  const std::string bad = packed_lengths("x_offsets", "samples", n, x_offsets, 1, x_len);
  if (!bad.empty()) return bad;
  f_off->assign(1, 0);
  for (int u = 0; u < n; ++u) f_off->push_back(f_off->back() + frames_for(fs, (*x_len)[u], frame_period));
  return "";
}

// ---- the CheapTrick, D4C and StoneMask stage calls: one plan, then load_batch and the stage's run
// EINVAL with last_error "<stage>: <what>", and " (utterance u)" for u >= 0
static const char *stage_name(StageKind stage) {
  return stage == STAGE_CHEAPTRICK ? "CheapTrick" : stage == STAGE_D4C ? "D4C" : "StoneMask";
}
static int stage_fail(Ctx *c, StageKind stage, const std::string &what, int u = -1) {
  c->last_error = std::string(stage_name(stage)) + ": " + what;
  if (u >= 0) c->last_error += " (utterance " + std::to_string(u) + ")";
  return WORLD_B200_EINVAL;
}

namespace wb {
int stage_plan(Ctx *c, const StageRequest &r, StagePlan *p) {
  const int n = r.n;
  auto fail = [&](const std::string &what, int u = -1) { return stage_fail(c, r.stage, what, u); };
  if (n < 0 || r.fs <= 0) return fail("n_utts must be >= 0 and fs > 0");
  if (r.stage == STAGE_STONEMASK && !stonemask_fits(r.fs))
    return fail("sampling rate too high for the twiddle table (fs <= 48000 supported)");
  if (r.stage == STAGE_D4C && !d4c_fits(r.fs)) return fail("sampling rate too high for the on-chip FFT (fft > 8192)");
  p->coded = r.coded;
  if (r.stage != STAGE_STONEMASK) {
    // one option for every utterance, or one each (then named in the messages)
    const bool ct = r.stage == STAGE_CHEAPTRICK;
    if ((ct ? !r.ct : !r.fft_size || !r.d4c) && (n > 0 || !r.per_utt)) return fail("the option must be given");
    p->fft_size.resize(n);
    p->q.resize(n);
    for (int u = 0; u < n; ++u) {
      const int k = r.per_utt ? u : 0;
      p->fft_size[u] = ct ? r.ct[k].fft_size : r.fft_size[k];
      p->q[u] = ct ? r.ct[k].q1 : r.d4c[k].threshold;
    }
    for (int u = 0; u < n; ++u) {
      const int f = p->fft_size[u], named = r.per_utt ? u : -1;
      if (ct && (f < 16 || f > WB_TW_N || (f & (f - 1))))
        return fail("fft_size must be a power of two in [16, 8192]", named);
      if (!ct && f < 4) return fail("fft_size must be at least 4", named);
      if (!std::isfinite(p->q[u])) return fail(ct ? "q1 must be finite" : "threshold must be finite", named);
    }
    p->row = r.row_stride || r.per_utt || n == 0 ? r.row_stride : p->fft_size[0] / 2 + 1;
    for (int u = 0; u < n && r.x_offsets && !r.row_stride; ++u) p->row = imax(p->row, p->fft_size[u] / 2 + 1);
    for (int u = 0; u < n && !r.coded; ++u)
      if (p->row < p->fft_size[u] / 2 + 1)
        return fail("row_stride is smaller than fft_size / 2 + 1", r.per_utt ? u : -1);
    p->table.assign(r.coded ? n : 0, -1);
    std::vector<int> first;   // coded: the first utterance of each table
    for (int u = 0; u < n && r.coded; ++u) {
      for (int t = 0; t < (int)first.size() && p->table[u] < 0; ++t)
        if (p->fft_size[first[t]] == p->fft_size[u]) p->table[u] = t;
      if (p->table[u] >= 0) continue;
      p->table[u] = (int)first.size();
      first.push_back(u);
      p->tables.emplace_back();
      const int rc = ct ? codec_sp_tables(c, r.fs, p->fft_size[u], r.dims, &p->tables.back())
                        : codec_ap_tables(c, r.fs, p->fft_size[u], &p->tables.back());
      if (rc) return fail(c->last_error, r.per_utt ? u : -1);
    }
    p->nothing = r.coded && !ct && GetNumberOfAperiodicities(r.fs) == 0;
  }
  if (r.x_offsets || r.f_offsets) {
    std::string bad = packed_lengths("x_offsets", "samples", n, r.x_offsets, 1, &p->x_len);
    if (bad.empty()) bad = packed_lengths("f_offsets", "frames", n, r.f_offsets, 0, &p->f_len);
    if (!bad.empty()) return fail(bad);
    p->x_off.assign(r.x_offsets, r.x_offsets + n + 1);
    p->f_off.assign(r.f_offsets, r.f_offsets + n + 1);
    return 0;
  }
  const char *who = stage_name(r.stage);
  int rc = row_lengths(c, who, "x", r.x_lengths, n, r.x_stride, 1, &p->x_len);
  if (!rc) rc = row_lengths(c, who, "f0", r.f0_lengths, n, r.f0_stride, 0, &p->f_len);
  return rc;
}
}  // namespace wb

// A stage entry point: x / time_axis / f0 / out are its device rows.
static int stage_batch(WorldB200 *h, const StageRequest &r, const double *x, const double *time_axis, const double *f0,
                       double *out) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *c = &h->c;
  if (!x || !time_axis || !f0) return stage_fail(c, r.stage, "x, time_axis and f0 must be given");
  StagePlan p;
  int rc = stage_plan(c, r, &p);
  if (rc || p.nothing) return rc;   // nothing to write below 12 kHz, like the reference's empty loops
  if (!out) return stage_fail(c, r.stage, "the output rows must be given");
  if (r.n == 0) return 0;
  Batch b;
  rc = load_batch(h, x, r.n, r.x_stride, p.x_len.data(), r.fs, time_axis, f0, p.f_len.data(), r.f0_stride, &b);
  if (rc) return rc;
  return r.stage == STAGE_CHEAPTRICK ? cheaptrick_run(c, p, b, 0, out)
         : r.stage == STAGE_D4C     ? d4c_run(c, p, b, 0, out)
                                    : stonemask_run(c, b, out);
}

extern "C" {

int world_b200_cheaptrick_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                                int f0_stride, const CheapTrickOption *opt, double *spectrogram) {
  StageRequest r{STAGE_CHEAPTRICK, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.ct = opt;
  return stage_batch(h, r, x, time_axis, f0, spectrogram);
}

int world_b200_d4c_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                         const double *time_axis, const double *f0, const int *f0_lengths, int f0_stride,
                         int fft_size, const D4COption *opt, double *aperiodicity) {
  StageRequest r{STAGE_D4C, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.fft_size = &fft_size; r.d4c = opt;
  return stage_batch(h, r, x, time_axis, f0, aperiodicity);
}

int world_b200_cheaptrick_coded_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                      int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                                      int f0_stride, const CheapTrickOption *opt, int number_of_dimensions,
                                      double *coded_spectral_envelope) {
  StageRequest r{STAGE_CHEAPTRICK, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.ct = opt; r.coded = true; r.dims = number_of_dimensions;
  return stage_batch(h, r, x, time_axis, f0, coded_spectral_envelope);
}

int world_b200_d4c_coded_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                               const double *time_axis, const double *f0, const int *f0_lengths, int f0_stride,
                               int fft_size, const D4COption *opt, double *coded_aperiodicity) {
  StageRequest r{STAGE_D4C, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.fft_size = &fft_size; r.d4c = opt; r.coded = true;
  return stage_batch(h, r, x, time_axis, f0, coded_aperiodicity);
}

int world_b200_cheaptrick_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                        int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                                        int f0_stride, const CheapTrickOption *options, int row_stride,
                                        double *spectrogram) {
  StageRequest r{STAGE_CHEAPTRICK, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.per_utt = true; r.ct = options; r.row_stride = row_stride;
  return stage_batch(h, r, x, time_axis, f0, spectrogram);
}

int world_b200_cheaptrick_coded_batch_options(WorldB200 *h, const double *x, int n, int x_stride,
                                              const int *x_lengths, int fs, const double *time_axis,
                                              const double *f0, const int *f0_lengths, int f0_stride,
                                              const CheapTrickOption *options, int number_of_dimensions,
                                              double *coded_spectral_envelope) {
  StageRequest r{STAGE_CHEAPTRICK, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.per_utt = true; r.ct = options; r.coded = true; r.dims = number_of_dimensions;
  return stage_batch(h, r, x, time_axis, f0, coded_spectral_envelope);
}

int world_b200_d4c_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                 const double *time_axis, const double *f0, const int *f0_lengths, int f0_stride,
                                 const int *fft_sizes, const D4COption *options, int row_stride,
                                 double *aperiodicity) {
  StageRequest r{STAGE_D4C, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.per_utt = true; r.fft_size = fft_sizes; r.d4c = options; r.row_stride = row_stride;
  return stage_batch(h, r, x, time_axis, f0, aperiodicity);
}

int world_b200_d4c_coded_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                       int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                                       int f0_stride, const int *fft_sizes, const D4COption *options,
                                       double *coded_aperiodicity) {
  StageRequest r{STAGE_D4C, n, x_stride, x_lengths, fs, f0_lengths, f0_stride};
  r.per_utt = true; r.fft_size = fft_sizes; r.d4c = options; r.coded = true;
  return stage_batch(h, r, x, time_axis, f0, coded_aperiodicity);
}

int world_b200_stonemask_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                               int fs, const double *time_axis, const double *f0, const int *f0_lengths,
                               int f0_stride, double *refined_f0) {
  return stage_batch(h, {STAGE_STONEMASK, n, x_stride, x_lengths, fs, f0_lengths, f0_stride}, x, time_axis, f0,
                     refined_f0);
}

}  // extern "C"

// A packed stage call: x [X], time_axis / f0 [F] and out [F][the planned row] read and written where they are.  The
// utterances run in chunks of consecutive utterances whose per-frame scratch fits the budget (and of at most 65535, the
// frame kernels' grid), each loaded with offsets relative to its first sample and frame.
static int stage_packed(WorldB200 *h, StageRequest r, const long long *x_offsets, const long long *f_offsets,
                        const double *x, const double *time_axis, const double *f0, double *out) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *c = &h->c;
  r.per_utt = true; r.x_offsets = x_offsets; r.f_offsets = f_offsets;
  StagePlan p;
  int rc = stage_plan(c, r, &p);
  if (rc) return rc;
  // empty arrays may be NULL: a batch without utterances or frames reads and writes nothing
  const bool frames = r.n > 0 && p.f_off[r.n] > 0;
  if ((r.n > 0 && !x) || (frames && (!time_axis || !f0)))
    return stage_fail(c, r.stage, "x, time_axis and f0 must be given");
  if (p.nothing) return 0;   // nothing to write below 12 kHz, like the reference's empty loops
  if (!out && frames) return stage_fail(c, r.stage, "the output rows must be given");
  const size_t row = r.stage == STAGE_STONEMASK                     ? 1
                     : !r.coded                                     ? (size_t)p.row
                     : r.stage == STAGE_CHEAPTRICK                  ? (size_t)r.dims
                                                                    : (size_t)GetNumberOfAperiodicities(r.fs);
  const long long *xo = p.x_off.data(), *fo = p.f_off.data();
  std::vector<long long> offs;
  for (int a = 0; a < r.n && !rc;) {
    int e = a, most_x = 1, most_f = 1;
    size_t bytes = 0;
    while (e < r.n && e - a < 65535) {
      const size_t more = WB_STAGE_UTT_BYTES + (size_t)p.f_len[e] * WB_STAGE_FRAME_BYTES;
      if (e > a && (WB_STAGE_CHUNK_BYTES + bytes + more > c->scratch_budget || fo[e + 1] - fo[a] > INT_MAX)) break;
      bytes += more;
      most_x = imax(most_x, p.x_len[e]);
      most_f = imax(most_f, p.f_len[e]);
      ++e;
    }
    const int m = e - a;
    offs.clear();
    for (int k = 0; k < m; ++k) offs.push_back(xo[a + k] - xo[a]);
    for (int k = 0; k <= m; ++k) offs.push_back(fo[a + k] - fo[a]);
    Batch b;
    rc = load_batch(h, x + xo[a], m, most_x, p.x_len.data() + a, r.fs, time_axis + fo[a], f0 + fo[a],
                    p.f_len.data() + a, most_f, &b, &offs);
    if (rc) break;
    b.f_off_host = offs.data() + m;
    double *o = out + (size_t)fo[a] * row;
    rc = r.stage == STAGE_CHEAPTRICK ? cheaptrick_run(c, p, b, a, o)
         : r.stage == STAGE_D4C     ? d4c_run(c, p, b, a, o)
                                    : stonemask_run(c, b, o);
    a = e;
  }
  return rc;
}

extern "C" {

int world_b200_stonemask_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs,
                                const double *time_axis, const double *f0, const long long *f_offsets,
                                double *refined_f0) {
  return stage_packed(h, {STAGE_STONEMASK, n, 0, nullptr, fs, nullptr, 0}, x_offsets, f_offsets, x, time_axis, f0,
                      refined_f0);
}

int world_b200_cheaptrick_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs,
                                 const double *time_axis, const double *f0, const long long *f_offsets,
                                 const CheapTrickOption *cheaptrick_options, int row_stride, double *spectrogram) {
  StageRequest r{STAGE_CHEAPTRICK, n, 0, nullptr, fs, nullptr, 0};
  r.ct = cheaptrick_options; r.row_stride = row_stride;
  return stage_packed(h, r, x_offsets, f_offsets, x, time_axis, f0, spectrogram);
}

int world_b200_cheaptrick_coded_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs,
                                       const double *time_axis, const double *f0, const long long *f_offsets,
                                       const CheapTrickOption *cheaptrick_options, int number_of_dimensions,
                                       double *coded_spectral_envelope) {
  StageRequest r{STAGE_CHEAPTRICK, n, 0, nullptr, fs, nullptr, 0};
  r.ct = cheaptrick_options; r.coded = true; r.dims = number_of_dimensions;
  return stage_packed(h, r, x_offsets, f_offsets, x, time_axis, f0, coded_spectral_envelope);
}

// d4c_options NULL: InitializeD4COption for every utterance
static int d4c_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs, const double *time_axis,
                      const double *f0, const long long *f_offsets, const int *fft_sizes, const D4COption *d4c_options,
                      bool coded, int row_stride, double *out) {
  StageRequest r{STAGE_D4C, n, 0, nullptr, fs, nullptr, 0};
  std::vector<D4COption> defaults;
  if (!d4c_options && n > 0) {
    defaults.resize(n);
    for (D4COption &o : defaults) InitializeD4COption(&o);
    d4c_options = defaults.data();
  }
  r.fft_size = fft_sizes; r.d4c = d4c_options; r.coded = coded; r.row_stride = row_stride;
  return stage_packed(h, r, x_offsets, f_offsets, x, time_axis, f0, out);
}

int world_b200_d4c_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs,
                          const double *time_axis, const double *f0, const long long *f_offsets, const int *fft_sizes,
                          const D4COption *d4c_options, int row_stride, double *aperiodicity) {
  return d4c_packed(h, x, n, x_offsets, fs, time_axis, f0, f_offsets, fft_sizes, d4c_options, false, row_stride,
                    aperiodicity);
}

int world_b200_d4c_coded_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs,
                                const double *time_axis, const double *f0, const long long *f_offsets,
                                const int *fft_sizes, const D4COption *d4c_options, double *coded_aperiodicity) {
  return d4c_packed(h, x, n, x_offsets, fs, time_axis, f0, f_offsets, fft_sizes, d4c_options, true, 0,
                    coded_aperiodicity);
}

}  // extern "C"

namespace wb {
// chain_plan without the caller's prefix on last_error
static int chain_checks(Ctx *c, const ChainRequest &r, ChainPlan *p) {
  auto fail = [c](const std::string &what) {
    c->last_error = what;
    return WORLD_B200_EINVAL;
  };
  const WorldB200AnalysisOption *opt = r.opt;
  if (!r.x || !opt || r.n < 0 || r.fs <= 0 || (!r.packed && r.x_stride <= 0) || r.f0_stride < 0)
    return fail("x and option must be given, with n_utts >= 0, fs > 0 and positive strides");
  if (r.nbit != 0 && r.nbit != 8 && r.nbit != 16 && r.nbit != 24 && r.nbit != 32)
    return fail("nbit must be 0, 8, 16, 24 or 32");
  if (r.row_stride < 0) return fail("row_stride must be >= 0");
  const int n = r.n, fft_size = opt->cheaptrick.fft_size;
  const bool spectral_options = r.cheaptrick_options || r.d4c_options;
  if ((r.spectrogram || r.aperiodicity) && fft_size < 16) return fail("CheapTrick: fft_size must be at least 16");
  // with per-utterance spectral options each utterance's size bounds number_of_dimensions (its codec tables, below)
  if (r.coded && (r.dims < 1 || (!spectral_options && r.dims > fft_size / 4 + 1)))
    return fail("number_of_dimensions must be in [1, fft_size/4 + 1]");

  // per-utterance F0 options: of the chain's F0 method, one frame_period (and, for DIO, one speed) for the batch, and
  // every utterance's range against the on-chip limits
  const bool harvest = opt->f0_method == WORLD_B200_F0_HARVEST;
  if (r.harvest_options && r.dio_options) return fail("per-utterance options of both F0 methods");
  if (r.harvest_options && !harvest)
    return fail("per-utterance Harvest options need f0_method == WORLD_B200_F0_HARVEST");
  if (r.dio_options && opt->f0_method != WORLD_B200_F0_DIO_STONEMASK)
    return fail("per-utterance DIO options need f0_method == WORLD_B200_F0_DIO_STONEMASK");
  RangeGroups groups;
  int rc = r.harvest_options ? harvest_plan(c, r.fs, r.harvest_options, n, true, opt->harvest.frame_period, &groups)
           : r.dio_options   ? dio_plan(c, r.fs, r.dio_options, n, true, opt->dio.frame_period, opt->dio.speed, &groups)
                             : 0;
  if (rc) return rc;
  p->frame_period = harvest ? opt->harvest.frame_period : opt->dio.frame_period;
  if (!(p->frame_period > 0.0)) return fail("the F0 method's frame_period must be > 0");

  // packed: the lengths come from the offsets, and the stage plans see rows as long as the longest utterance
  int x_stride = r.x_stride;
  const int *x_lengths = r.x_lengths;
  if (r.packed) {
    const std::string bad = packed_layout(r.fs, n, r.x_offsets, p->frame_period, &p->x_len, &p->f_off);
    if (!bad.empty()) return fail(bad);
    x_stride = n ? *std::max_element(p->x_len.begin(), p->x_len.end()) : 1;
    x_lengths = p->x_len.data();
  }
  p->f_len.resize(n);
  int most = 1;
  for (int u = 0; u < n; ++u) {
    const int xl = x_lengths ? x_lengths[u] : x_stride;
    if (xl < 1 || xl > x_stride)
      return fail("x_lengths[" + std::to_string(u) + "] = " + std::to_string(xl) + " is outside its padded row of " +
                  std::to_string(x_stride) + " samples");
    p->f_len[u] = frames_for(r.fs, xl, p->frame_period);
    if (r.f0_stride && p->f_len[u] > r.f0_stride)
      return fail("f0_stride smaller than the frame count of an utterance (utterance " + std::to_string(u) + ")");
    most = imax(most, p->f_len[u]);
  }
  p->f0_stride = r.f0_stride ? r.f0_stride : most;

  // The stage plans: CheapTrick when a spectrogram is asked for, D4C when an aperiodicity is (a transform needs both),
  // StoneMask's sampling-rate limit for DIO.  Each utterance's CheapTrick option, and D4C's fft_size (its CheapTrick
  // size) and option, with the per-call option standing in for a NULL per-utterance array.
  const bool transform = r.transform;
  StageRequest s{STAGE_CHEAPTRICK, n, x_stride, x_lengths, r.fs, p->f_len.data(), p->f0_stride};
  s.ct = &opt->cheaptrick; s.fft_size = &opt->cheaptrick.fft_size; s.d4c = &opt->d4c;
  s.coded = r.coded; s.dims = r.dims;
  s.row_stride = r.coded ? 0 : r.row_stride;   // the stage plans check it against every utterance's size
  std::vector<CheapTrickOption> cts;
  std::vector<D4COption> d4s;
  std::vector<int> d4_fft;
  if (spectral_options) {
    cts.assign(n, opt->cheaptrick);
    d4s.assign(n, opt->d4c);
    if (r.cheaptrick_options) std::copy(r.cheaptrick_options, r.cheaptrick_options + n, cts.begin());
    if (r.d4c_options) std::copy(r.d4c_options, r.d4c_options + n, d4s.begin());
    for (const CheapTrickOption &o : cts) d4_fft.push_back(o.fft_size);
    s.per_utt = true; s.ct = cts.data(); s.fft_size = d4_fft.data(); s.d4c = d4s.data();
    // full rows without a caller's stride (a transform's): every utterance's row as wide as the largest size's
    if (!r.coded && !r.row_stride)
      for (const int f : d4_fft) s.row_stride = imax(s.row_stride, f / 2 + 1);
  }
  if ((r.spectrogram || transform) && (rc = stage_plan(c, s, &p->ct))) return rc;
  s.stage = STAGE_D4C;
  if ((r.aperiodicity || transform) && (rc = stage_plan(c, s, &p->d4))) return rc;
  s.stage = STAGE_STONEMASK;
  StagePlan stonemask;
  if (!harvest && (rc = stage_plan(c, s, &stonemask))) return rc;
  const size_t full_row = s.row_stride ? (size_t)s.row_stride : (size_t)(fft_size / 2 + 1);
  p->sp_row = r.coded ? (size_t)r.dims : full_row;
  p->ap_row = r.coded ? (size_t)GetNumberOfAperiodicities(r.fs) : full_row;
  p->want_sp = r.spectrogram != nullptr;
  p->want_ap = r.aperiodicity != nullptr && !p->d4.nothing;   // no bands below 12 kHz: D4C is skipped
  return 0;
}

int chain_plan(Ctx *c, const ChainRequest &r, const char *who, ChainPlan *p) {
  const int rc = chain_checks(c, r, p);
  if (rc) c->last_error = std::string(who) + ": " + c->last_error;
  return rc;
}

int chain_f0(WorldB200 *h, const ChainRequest &r, const ChainPlan &p, int u0, int m, const double *x, double *time_axis,
             double *f0, const PackedSlice *ps) {
  const WorldB200AnalysisOption *opt = r.opt;
  const int *xl = ps ? p.x_len.data() + u0 : r.x_lengths ? r.x_lengths + u0 : nullptr;
  const int x_stride = ps ? ps->x_stride : r.x_stride, f0_stride = ps ? ps->f0_stride : p.f0_stride;
  if (opt->f0_method == WORLD_B200_F0_HARVEST)
    return r.harvest_options ? world_b200_harvest_batch_options(h, x, m, x_stride, xl, r.fs, r.harvest_options + u0,
                                                                time_axis, f0, f0_stride)
                             : world_b200_harvest_batch(h, x, m, x_stride, xl, r.fs, &opt->harvest, time_axis, f0,
                                                        f0_stride);
  int rc = r.dio_options
               ? world_b200_dio_batch_options(h, x, m, x_stride, xl, r.fs, r.dio_options + u0, time_axis, f0, f0_stride)
               : world_b200_dio_batch(h, x, m, x_stride, xl, r.fs, &opt->dio, time_axis, f0, f0_stride);
  if (!rc)
    rc = world_b200_stonemask_batch(h, x, m, x_stride, xl, r.fs, time_axis, f0, p.f_len.data() + u0, f0_stride, f0);
  return rc;
}

int chain_spectral(WorldB200 *h, const ChainRequest &r, const ChainPlan &p, int u0, int m, const double *x,
                   const double *time_axis, const double *f0, double *sp, double *ap, const PackedSlice *ps) {
  if (!sp && !ap) return 0;
  const StagePlan &lens = sp ? p.ct : p.d4;   // both plans hold the chain's lengths
  Batch b;
  int rc = load_batch(h, x, m, ps ? ps->x_stride : r.x_stride, lens.x_len.data() + u0, r.fs, time_axis, f0,
                      lens.f_len.data() + u0, ps ? ps->f0_stride : p.f0_stride, &b);
  if (ps) b.f_off = ps->f_off;
  if (!rc && sp) rc = cheaptrick_run(&h->c, p.ct, b, u0, sp);
  if (!rc && ap) rc = d4c_run(&h->c, p.d4, b, u0, ap);
  return rc;
}
}  // namespace wb

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

// The F0 stage calls: opt is one option for every utterance, or (per_utt) an array of n.  The options are checked and
// grouped before the lengths are uploaded: a bad option queues nothing on the device.
template <class Option>
static int f0_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs, const Option *opt,
                    bool per_utt, double *time_axis, double *f0, int f0_stride) {
  if (!h || !x || !time_axis || !f0 || !opt || n < 0 || fs <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  constexpr bool harvest = std::is_same<Option, HarvestOption>::value;
  RangeGroups groups;
  int rc;
  if constexpr (harvest) rc = harvest_plan(&h->c, fs, opt, n, per_utt, opt->frame_period, &groups);
  else rc = dio_plan(&h->c, fs, opt, n, per_utt, opt->frame_period, opt->speed, &groups);
  if (rc) return rc;
  std::vector<int> xl, fl;
  rc = row_lengths(&h->c, harvest ? "Harvest" : "DIO", "x", x_lengths, n, x_stride, 1, &xl);
  if (!rc) rc = f0_lengths_from_x(n, x_stride, x_lengths, fs, opt->frame_period, f0_stride, &fl, &h->c.last_error);
  if (rc) return rc;
  Batch b;
  rc = load_batch(h, x, n, x_stride, xl.data(), fs, time_axis, f0, fl.data(), f0_stride, &b);
  if (rc) return rc;
  b.x_len_host = x_lengths;
  if constexpr (harvest) {
    std::vector<int> l1(n > 0 ? n : 1);
    for (int i = 0; i < n; ++i) l1[i] = frames_for(fs, x_lengths ? x_lengths[i] : x_stride, 1.0);
    b.l1_host = l1.data();
    return harvest_run(&h->c, b, opt->frame_period, groups, time_axis, f0);
  } else {
    return dio_run(&h->c, b, opt, per_utt, groups, time_axis, f0);
  }
}

extern "C" {

int world_b200_dio_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                         const DioOption *opt, double *time_axis, double *f0, int f0_stride) {
  return f0_batch(h, x, n, x_stride, x_lengths, fs, opt, false, time_axis, f0, f0_stride);
}

int world_b200_dio_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                 const DioOption *dio_options, double *time_axis, double *f0, int f0_stride) {
  return f0_batch(h, x, n, x_stride, x_lengths, fs, dio_options, true, time_axis, f0, f0_stride);
}

int world_b200_harvest_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                             int fs, const HarvestOption *opt, double *time_axis, double *f0, int f0_stride) {
  return f0_batch(h, x, n, x_stride, x_lengths, fs, opt, false, time_axis, f0, f0_stride);
}

int world_b200_harvest_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                     const HarvestOption *harvest_options, double *time_axis, double *f0,
                                     int f0_stride) {
  return f0_batch(h, x, n, x_stride, x_lengths, fs, harvest_options, true, time_axis, f0, f0_stride);
}

}  // extern "C"

namespace {

// The two lanes of a chain cut into slices: sibling contexts on their own non-blocking streams (created on first use),
// ordered after the work already on the context's stream, each with half the context's scratch budget and one pooled
// buffer sized for the largest of its slices.  Slices alternate between the lanes.  The chain has one lane, the context
// itself, when it is one slice (and always on the host emulation, which has one stream).  On every return path the
// destructor makes the context's stream wait for both lanes, gives the buffers back and restores the context's budget.
class LaneScope {
 public:
  explicit LaneScope(WorldB200 *h) : h_(h), own_budget_(h->c.scratch_budget) { lanes_[0] = lanes_[1] = h; }
  LaneScope(const LaneScope &) = delete;
  LaneScope &operator=(const LaneScope &) = delete;
  // bounds: the n_slices + 1 slice boundaries; bytes(s): the buffer slice s needs (0: none), and a lane's buffer is
  // the largest of its slices'.  A buffer comes from its lane's pool, not its arena (the stage drivers reset the arena
  // when they return), and its bytes come out of the lane's scratch budget; the stages keep at least half of that
  // budget (less would only mean more passes).
  template <class Bytes>
  int open(const std::vector<int> &bounds, Bytes bytes) {
    const int n_slices = (int)bounds.size() - 1;
#ifndef WB_EMU
    if (n_slices > 1) {
      WorldB200 *two[2];
      for (int l = 0; l < 2; ++l) {
        if (!h_->lane[l]) {
          int rc = world_b200_create(h_->c.device, &h_->lane[l]);
          if (rc) { h_->c.last_error = "analyze_batch: cannot create a lane context"; return rc; }
          cudaStream_t st;
          cudaEvent_t ev;
          // equal (lowest) priority for both lanes: giving one lane the highest priority was measured slower;
          // only the communication stream outranks them (wb_multi.cu)
          if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess ||
              cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
            h_->c.last_error = "analyze_batch: cannot create a lane stream";
            return WORLD_B200_ECUDA;
          }
          h_->lane_stream[l] = st; h_->ev_join[l] = ev;
          h_->lane[l]->c.stream = st;
        }
        h_->lane[l]->c.scratch_budget = h_->c.scratch_budget / 2;
        two[l] = h_->lane[l];
      }
      if (!h_->ev_fork) {
        cudaEvent_t ev;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return WORLD_B200_ECUDA;
        h_->ev_fork = ev;
      }
      cudaEventRecord((cudaEvent_t)h_->ev_fork, h_->c.stream);
      for (int l = 0; l < 2; ++l) cudaStreamWaitEvent((cudaStream_t)h_->lane_stream[l], (cudaEvent_t)h_->ev_fork, 0);
      lanes_[0] = two[0]; lanes_[1] = two[1];
    }
#endif
    size_t lane_bytes[2] = {0, 0};
    for (int s = 0; s < n_slices; ++s) {
      most_[index(s)] = imax(most_[index(s)], bounds[s + 1] - bounds[s]);
      lane_bytes[index(s)] = std::max(lane_bytes[index(s)], (size_t)bytes(s));
    }
    for (int l = 0; l < (one_lane() ? 1 : 2); ++l) {
      const size_t b = lane_bytes[l];
      if (b == 0) continue;
      Ctx *c = &lanes_[l]->c;
      buf_[l] = (unsigned char *)pool_acquire(c, b);
      if (!buf_[l]) { h_->c.last_error = c->last_error; return WORLD_B200_ENOMEM; }
      c->scratch_budget -= b < c->scratch_budget / 2 ? b : c->scratch_budget / 2;
    }
    return 0;
  }
  ~LaneScope() {
#ifndef WB_EMU
    if (!one_lane())   // even after an error: the caller's stream must not run ahead of the lanes
      for (int l = 0; l < 2; ++l) {
        cudaEventRecord((cudaEvent_t)h_->ev_join[l], (cudaStream_t)h_->lane_stream[l]);
        cudaStreamWaitEvent(h_->c.stream, (cudaEvent_t)h_->ev_join[l], 0);
      }
#endif
    // back to the pools while the lanes may still read them: a pooled buffer is only handed out again to work that is
    // ordered after this call's (the lane's next slices, or the host pipelines, whose uploads wait for the stream)
    for (int l = 0; l < 2; ++l) pool_release(&lanes_[l]->c, buf_[l]);
    h_->c.scratch_budget = own_budget_;
  }
  bool one_lane() const { return lanes_[0] == lanes_[1]; }
  WorldB200 *lane(int s) const { return lanes_[index(s)]; }          // slice s's lane
  unsigned char *buffer(int s) const { return buf_[index(s)]; }      // ... its buffer
  int most(int s) const { return most_[index(s)]; }                  // ... and the largest slice of that lane

 private:
  int index(int s) const { return one_lane() ? 0 : (s & 1); }
  WorldB200 *h_;
  WorldB200 *lanes_[2];
  unsigned char *buf_[2] = {nullptr, nullptr};
  int most_[2] = {0, 0};
  size_t own_budget_;
};

}  // namespace

extern "C" {

// The whole chain on device arrays, cut into utterance slices that alternate between two lanes (sibling contexts
// on their own non-blocking streams).  Per slice the stages run in order on the lane's stream; the two lanes run
// concurrently, so the latency-bound per-utterance kernels of one slice (contour tracking, candidate clean-up, the
// draw stream, decimation) execute under the FP64-bound kernels of the other.  Ordered after the work already on the
// context's stream; that stream waits for both lanes before the function returns (no host synchronisation).
// gather = false: time_axis / f0 / spectrogram / aperiodicity hold this call's n utterances.
// gather = true (multi-GPU): they are the FULL arrays of n_ranks * n utterances; this rank computes into block `rank`
// and every finished slice is broadcast to the other ranks on the communication stream while the next one is computed.
// PCM input (nbit != 0) is converted slice by slice on the lane that analyses it; the per-utterance option arrays are
// split with the utterances.
static int analyze_chain(WorldB200 *h, const ChainRequest &r, bool gather) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  const char *who = r.coded ? "analyze_coded_batch" : "analyze_batch";
  if (!r.time_axis || !r.f0 || r.f0_stride <= 0) {
    h->c.last_error = std::string(who) + ": time_axis and f0 must be given, with f0_stride > 0";
    return WORLD_B200_EINVAL;
  }
  ChainPlan p;
  int rc = chain_plan(&h->c, r, who, &p);
  if (rc || r.n == 0) return rc;
  const int n = r.n, nbit = r.nbit, x_stride = r.x_stride, f0_stride = p.f0_stride;
  const size_t sp_row = p.sp_row, ap_row = p.ap_row;
  double *time_axis = r.time_axis, *f0 = r.f0;
  double *spectrogram = p.want_sp ? r.spectrogram : nullptr, *aperiodicity = p.want_ap ? r.aperiodicity : nullptr;
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
  // nbit != 0: each lane converts its slice into a float64 buffer, which the slice's three stages then read.  A lane
  // runs its slices in stream order, so one buffer per lane, sized for its largest slice, serves all of them.
  LaneScope lanes(h);
  rc = lanes.open(bounds, [&](int s) {
    return nbit ? (size_t)(bounds[s + 1] - bounds[s]) * x_stride * sizeof(double) : (size_t)0;
  });
  if (rc) return rc;
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
  if (exchange && !getenv("WB_NO_P2P")) {
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
    WorldB200 *L = lanes.lane(s);
    const double *xs = (const double *)lanes.buffer(s);
    if (nbit)
      rc = world_b200_pcm_to_double_batch(L, (const unsigned char *)r.x + (size_t)u0 * x_stride * (nbit / 8), nbit, m,
                                          x_stride, r.x_lengths ? r.x_lengths + u0 : nullptr, (double *)lanes.buffer(s));
    else
      xs = (const double *)r.x + (size_t)u0 * x_stride;
    double *ts = time_axis + (size_t)u0 * f0_stride, *fs_ = f0 + (size_t)u0 * f0_stride;
    if (!rc) rc = chain_f0(L, r, p, u0, m, xs, ts, fs_);
    if (!rc)
      rc = chain_spectral(L, r, p, u0, m, xs, ts, fs_, spectrogram ? spectrogram + (size_t)u0 * f0_stride * sp_row : nullptr,
                          aperiodicity ? aperiodicity + (size_t)u0 * f0_stride * ap_row : nullptr);
    if (rc && L != h) h->c.last_error = L->c.last_error;
#ifndef WB_EMU
    if (!rc && exchange) {
      // rows u0..u1 of every rank's block, as soon as this rank's are final (event on the lane's stream)
      while (!rc && (int)h->ev_slice.size() <= s) {
        cudaEvent_t ev;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess) h->ev_slice.push_back(ev);
        else { h->c.last_error = "cudaEventCreate failed"; rc = WORLD_B200_ECUDA; }
      }
      if (!rc) {
        cudaEvent_t ev = (cudaEvent_t)h->ev_slice[s];
        cudaEventRecord(ev, L->c.stream);
        std::string err;
        const int g = push ? comm_p2p_push(h->comm, 4, full_elems, (size_t)n, (size_t)u0, (size_t)m, ev, &err)
                           : comm_gather_rows_multi(h->comm, 4, fulls, full_elems, (size_t)n, (size_t)u0, (size_t)m, ev, &err);
        if (g) { h->c.last_error = err; rc = WORLD_B200_ECUDA; }
      }
    }
#endif
  }
#ifndef WB_EMU
  if (exchange) {
    std::string err;
    const int g = push ? comm_p2p_finish(h->comm, h->c.stream, &err) : comm_join(h->comm, h->c.stream, &err);
    if (g && !rc) { h->c.last_error = err; rc = WORLD_B200_ECUDA; }
  }
#endif
  return rc;
}

}  // extern "C"

// A packed slice's time axis and f0, from the lane's padded rows (f_stride frames) to the packed rows: utterance u
// (blockIdx.y) has f_off[u + 1] - f_off[u] frames, written from row f_off[u].  t_out NULL: f0 only (a transform).
WB_KERNEL_PLAIN scatter_f0_kernel(const long long *__restrict__ f_off, int f_stride, const double *__restrict__ t,
                                  const double *__restrict__ f, double *__restrict__ t_out, double *__restrict__ f_out) {
  const int u = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long at = f_off[u] + i;
  if (at >= f_off[u + 1]) return;
  if (t_out) t_out[at] = t[(size_t)u * f_stride + i];
  f_out[at] = f[(size_t)u * f_stride + i];
}

namespace wb {

// Lane slices of the packed utterances [c0, c1): n_slices cuts at equal shares of their samples, so that both lanes get
// equal work, then halved (at the middle sample) until each slice's padded rows -- bytes(u0, u1) -- fit `cap`, or the
// slice is one utterance.  Padded rows are as long as a slice's longest utterance: one long utterance among many short
// ones would otherwise pad them all.
template <class Bytes>
static std::vector<int> packed_bounds(const long long *x_offsets, int c0, int c1, int n_slices, size_t cap,
                                      Bytes bytes) {
  std::vector<int> bounds{c0};
  const long long base = x_offsets[c0], total = x_offsets[c1] - base;
  // the first utterance at or past sample `at` of [u0, u1], kept inside (u0, u1)
  auto cut = [&](int u0, int u1, long long at) {
    const int u = (int)(std::lower_bound(x_offsets + u0, x_offsets + u1, at) - x_offsets);
    return imin(u1 - 1, imax(u0 + 1, u));
  };
  std::vector<int> stack;
  for (int s = 0; s < n_slices; ++s) {
    const int u1 = s + 1 == n_slices ? c1 : cut(bounds.back(), c1, base + total * (s + 1) / n_slices);
    if (u1 <= bounds.back()) continue;
    stack.assign(1, u1);
    while (!stack.empty()) {   // halve [bounds.back(), stack.back()) until it fits
      const int u0 = bounds.back(), e = stack.back();
      if (e - u0 > 1 && bytes(u0, e) > cap) {
        stack.push_back(cut(u0, e, (x_offsets[u0] + x_offsets[e]) / 2));
      } else {
        bounds.push_back(e);
        stack.pop_back();
      }
    }
  }
  return bounds;
}

int packed_run(WorldB200 *h, const ChainRequest &r, const ChainPlan &p, int c0, int c1, const void *x,
               double *time_axis, double *f0, double *sp, double *ap) {
  const long long *xo = r.x_offsets;
  const long long *fo = p.f_off.data();
  // a slice's lane buffer: its x and f0 offsets, then its padded rows of samples, time axis and f0
  struct Rows { int x_stride, f0_stride; size_t off, x, t, f, total; };
  auto rows_of = [&](int u0, int u1) {
    Rows w{1, 1, 0, 0, 0, 0, 0};
    for (int u = u0; u < u1; ++u) { w.x_stride = imax(w.x_stride, p.x_len[u]); w.f0_stride = imax(w.f0_stride, p.f_len[u]); }
    const size_t m = (size_t)(u1 - u0);
    w.x = 16 * (m + 1);
    w.t = w.x + m * w.x_stride * 8;
    w.f = w.t + m * w.f0_stride * 8;
    w.total = w.f + m * w.f0_stride * 8;
    return w;
  };
  int n_slices = 2;
  if (const char *e = getenv("WB_LANE_SLICES")) n_slices = atoi(e);
  n_slices = imax(1, imin(n_slices, c1 - c0));
  // each lane's buffer comes out of its half of the budget, and the stages keep at least half of that
  const std::vector<int> bounds = packed_bounds(xo, c0, c1, n_slices, h->c.scratch_budget / 4,
                                                [&](int u0, int u1) { return rows_of(u0, u1).total; });
  LaneScope lanes(h);
  int rc = lanes.open(bounds, [&](int s) { return rows_of(bounds[s], bounds[s + 1]).total; });
  std::vector<long long> offs;
  for (size_t s = 0; s + 1 < bounds.size() && !rc; ++s) {
    const int u0 = bounds[s], m = bounds[s + 1] - u0;
    WorldB200 *L = lanes.lane((int)s);
    Ctx *lc = &L->c;
    const Rows w = rows_of(u0, u0 + m);
    unsigned char *buf = lanes.buffer((int)s);
    // offsets relative to x and to the output rows
    offs.resize(2 * ((size_t)m + 1));
    for (int k = 0; k <= m; ++k) { offs[k] = xo[u0 + k] - xo[c0]; offs[m + 1 + k] = fo[u0 + k] - fo[c0]; }
    const long long *x_off = (const long long *)buf, *f_off = x_off + m + 1;
    double *xs = (double *)(buf + w.x), *ts = (double *)(buf + w.t), *fs_ = (double *)(buf + w.f);
    rc = dev_memcpy_h2d(lc, buf, offs.data(), offs.size() * 8);
    if (!rc) rc = gather_samples(lc, x, r.nbit, x_off, m, w.x_stride, w.x_stride, xs);
    const PackedSlice ps{w.x_stride, w.f0_stride, f_off};
    if (!rc) rc = chain_f0(L, r, p, u0, m, xs, ts, fs_, &ps);
    if (!rc) rc = chain_spectral(L, r, p, u0, m, xs, ts, fs_, sp, ap, &ps);
    for (int k0 = 0; k0 < m && !rc; k0 += 65535) {
      WB_LAUNCH_FLAT(scatter_f0_kernel, dim3((unsigned)((w.f0_stride + 255) / 256), (unsigned)imin(65535, m - k0)), 256,
                     0, lc->stream, f_off + k0, w.f0_stride, ts + (size_t)k0 * w.f0_stride,
                     fs_ + (size_t)k0 * w.f0_stride, time_axis, f0);
      rc = dev_check(lc, "packed f0");
    }
    if (rc && L != h) h->c.last_error = L->c.last_error;
  }
  return rc;
}

}  // namespace wb

extern "C" {

int world_b200_analyze_batch(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                             const WorldB200AnalysisOption *opt, double *time_axis, double *f0, int f0_stride,
                             double *spectrogram, double *aperiodicity) {
  return analyze_chain(h, ChainRequest(x, 0, n, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram,
                                       aperiodicity), false);
}

int world_b200_analyze_batch_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs,
                                     const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                     double *time_axis, double *f0, int f0_stride, double *spectrogram,
                                     double *aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  ChainRequest r(x, 0, n, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram, aperiodicity);
  r.harvest_options = harvest_options;
  return analyze_chain(h, r, false);
}

int world_b200_analyze_batch_dio_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                         int fs, const WorldB200AnalysisOption *opt, const DioOption *dio_options,
                                         double *time_axis, double *f0, int f0_stride, double *spectrogram,
                                         double *aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  ChainRequest r(x, 0, n, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram, aperiodicity);
  r.dio_options = dio_options;
  return analyze_chain(h, r, false);
}

int world_b200_analyze_batch_spectral_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                              int fs, const WorldB200AnalysisOption *opt,
                                              const HarvestOption *harvest_options, const DioOption *dio_options,
                                              const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                              double *time_axis, double *f0, int f0_stride, int row_stride,
                                              double *spectrogram, double *aperiodicity) {
  ChainRequest r(x, 0, n, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram, aperiodicity);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options; r.row_stride = row_stride;
  return analyze_chain(h, r, false);
}

}  // extern "C"

// ---- voice transformation: analysis, modification and synthesis in one call (world_b200_transform_*)
namespace wb {

// Every check of the call before any work is queued (EINVAL, last_error naming the first bad utterance): y, nbit_out,
// the analysis plan and time_scale here, then the synthesis plan of the analysis rows.
int transform_check(WorldB200 *h, const ChainRequest &r, const double *f0_scale, const double *spectral_ratio,
                    const double *time_scale, int nbit_out, void *y, int y_stride, const char *who, TransformPlan *tp) {
  Ctx *c = &h->c;
  auto fail = [&](const char *what) {
    c->last_error = std::string(who) + ": " + what;
    return WORLD_B200_EINVAL;
  };
  if (!y || (!r.packed && y_stride <= 0)) return fail(r.packed ? "y must be given" : "y must be given, with y_stride > 0");
  if (nbit_out != 0 && nbit_out != 16) return fail("nbit_out must be 0 (float64) or 16 (int16)");
  const ChainPlan &p = tp->chain;
  const int rc = chain_plan(c, r, who, &tp->chain);
  if (rc) return rc;
  std::vector<int> y_len(r.n);
  std::vector<double> fp(r.n);
  std::vector<long long> y_off(1, 0);
  for (int u = 0; u < r.n; ++u) {
    const double ts = time_scale ? time_scale[u] : 1.0;
    char msg[256];
    if (!(ts > 0.0) || !isfinite(ts)) {
      snprintf(msg, sizeof msg, "time_scale[%d] = %.17g is not a finite factor > 0", u, ts);
      return fail(msg);
    }
    const int x_len = r.packed ? p.x_len[u] : r.x_lengths ? r.x_lengths[u] : r.x_stride;
    y_len[u] = world_b200_transform_samples(r.fs, x_len, p.frame_period, ts);
    fp[u] = (p.frame_period * ts) / 1000.0;   // synthesis_batch's frame_period / 1000.0, with the same product
    if (r.packed && y_len[u] == 0) {
      snprintf(msg, sizeof msg, "the output of utterance %d (%d samples at time_scale %.17g) does not fit an int", u,
               x_len, ts);
      return fail(msg);
    }
    y_off.push_back(y_off.back() + y_len[u]);
  }
  SynthesisRequest s{nullptr, p.f_len.data(), r.n, p.f0_stride, nullptr, nullptr, r.opt->cheaptrick.fft_size,
                     p.frame_period, r.fs, y_len.data(), y_stride, y, nbit_out};
  s.f0_scale = f0_scale; s.spectral_ratio = spectral_ratio; s.transform = true; s.fp = fp.data();
  if (r.cheaptrick_options || r.d4c_options || r.packed) {   // each utterance synthesised at its CheapTrick size
    s.per_utt = true; s.fft_sizes = p.ct.fft_size.data(); s.row_stride = (int)p.sp_row;
  }
  if (r.packed) { s.f_offsets = p.f_off.data(); s.y_offsets = y_off.data(); }
  return synthesis_plan(c, s, who, &tp->syn);
}

// The slice loop of both transform drivers.  Slice s is utterances [bounds[s], bounds[s + 1]) and bytes(s) the rows it
// keeps in its lane's buffer from its analysis to its synthesis; analyse(lanes, s) and synthesise(lanes, s) enqueue its
// two halves on lanes.lane(s).  Issue order A(0), A(1), S(0), A(2), S(1), ... (A = F0 stage, CheapTrick, D4C and
// modify; S = synthesis): a lane runs its slices in stream order, so A(s + 1) never overwrites rows S(s - 1) still
// reads, and while synthesis_run waits for its pulse counts (a host synchronisation of its lane), the other lane has an
// analysis queued.  One lane (one slice, or the host emulation) runs A(s), S(s) in turn.  The caller's stream waits for
// both lanes on return.
template <class Bytes, class Analyse, class Synthesise>
static int transform_slices(WorldB200 *h, const std::vector<int> &bounds, Bytes bytes, Analyse analyse,
                            Synthesise synthesise) {
  const int n_slices = (int)bounds.size() - 1;
  LaneScope lanes(h);
  int rc = lanes.open(bounds, bytes);
  if (rc) return rc;
  const int lag = lanes.one_lane() ? 0 : 1;
  for (int k = 0; k < n_slices + lag && !rc; ++k) {
    if (k < n_slices) rc = analyse(lanes, k);
    if (!rc && k >= lag) rc = synthesise(lanes, k - lag);
  }
  return rc;
}

// A lane's error as the context's
static int lane_error(WorldB200 *h, WorldB200 *L, int e) {
  if (e && L != h) h->c.last_error = L->c.last_error;
  return e;
}

// The packed transform over utterances [u0, u0 + n): x at sample x_offsets[u0] and y at sample y_off[u0] (DEVICE).
// Slices are cut by packed_bounds at equal shares of the samples, halved until a slice's own rows fit half its lane's
// budget.  A slice's lane buffer holds its offsets, padded rows of samples, time axis and f0 as long as its longest
// utterance (what the F0 stage reads), then its packed f0, spectrogram and aperiodicity frames (what CheapTrick and D4C
// write and modification and synthesis read), so one long utterance only lengthens the rows of its own slice.
static int transform_packed_run(WorldB200 *h, const ChainRequest &r, const TransformPlan &tp, const void *x, int u0,
                                int n, void *y, const ModifyCurves *cv) {
  const ChainPlan &p = tp.chain;
  const long long *xo = r.x_offsets, *fo = p.f_off.data(), *yo = tp.syn.y_off.data();
  const size_t row = p.sp_row, out_bytes = tp.syn.nbit ? 2 : 8;
  struct Rows { int x_stride, f0_stride; size_t x, t, f, pf, sp, ap, total; };
  auto rows_of = [&](int a, int b) {
    Rows w{1, 1, 0, 0, 0, 0, 0, 0, 0};
    for (int u = a; u < b; ++u) { w.x_stride = imax(w.x_stride, p.x_len[u]); w.f0_stride = imax(w.f0_stride, p.f_len[u]); }
    const size_t m = (size_t)(b - a), frames = (size_t)(fo[b] - fo[a]);
    ArenaPlan l;
    l.add(16 * (m + 1));
    w.x = l.add(m * w.x_stride * 8);
    w.t = l.add(m * w.f0_stride * 8); w.f = l.add(m * w.f0_stride * 8);
    w.pf = l.add(frames * 8); w.sp = l.add(frames * row * 8); w.ap = l.add(frames * row * 8);
    w.total = l.total;
    return w;
  };
#ifndef WB_EMU
  const bool two = n > 1;
#else
  const bool two = false;
#endif
  const size_t cap = h->c.scratch_budget / (two ? 2 : 1) / 2;
  size_t own = 0;   // every utterance's rows on their own: the least the slices can take
  for (int u = u0; u < u0 + n; ++u) own += rows_of(u, u + 1).total;
  int n_slices = (int)std::min<size_t>((size_t)n, std::max<size_t>(1, (own + cap - 1) / cap));
  if (two) n_slices = imin(n, (n_slices + 1) / 2 * 2);   // an even count: both lanes get the same work
  const std::vector<int> bounds = packed_bounds(xo, u0, u0 + n, n_slices, cap,
                                                [&](int a, int b) { return rows_of(a, b).total; });
  auto bytes = [&](int s) { return rows_of(bounds[s], bounds[s + 1]).total; };
  std::vector<long long> offs;
  auto analyse = [&](const LaneScope &lanes, int s) {
    const int a = bounds[s], m = bounds[s + 1] - a;
    WorldB200 *L = lanes.lane(s);
    Ctx *lc = &L->c;
    const Rows w = rows_of(a, a + m);
    unsigned char *buf = lanes.buffer(s);
    // sample offsets relative to x, frame offsets relative to the slice's first frame
    offs.resize(2 * ((size_t)m + 1));
    for (int k = 0; k <= m; ++k) { offs[k] = xo[a + k] - xo[u0]; offs[m + 1 + k] = fo[a + k] - fo[a]; }
    const long long *x_off = (const long long *)buf, *f_off = x_off + m + 1;
    double *xs = (double *)(buf + w.x), *ts = (double *)(buf + w.t), *fs_ = (double *)(buf + w.f);
    double *f0 = (double *)(buf + w.pf), *sp = (double *)(buf + w.sp), *ap = (double *)(buf + w.ap);
    int e = dev_memcpy_h2d(lc, buf, offs.data(), offs.size() * 8);
    if (!e) e = gather_samples(lc, x, r.nbit, x_off, m, w.x_stride, w.x_stride, xs);
    const PackedSlice ps{w.x_stride, w.f0_stride, f_off};
    if (!e) e = chain_f0(L, r, p, a, m, xs, ts, fs_, &ps);
    if (!e) e = chain_spectral(L, r, p, a, m, xs, ts, fs_, sp, ap, &ps);
    for (int k0 = 0; k0 < m && !e; k0 += 65535) {
      WB_LAUNCH_FLAT(scatter_f0_kernel, dim3((unsigned)((w.f0_stride + 255) / 256), (unsigned)imin(65535, m - k0)), 256,
                     0, lc->stream, f_off + k0, w.f0_stride, ts + (size_t)k0 * w.f0_stride,
                     fs_ + (size_t)k0 * w.f0_stride, nullptr, f0);
      e = dev_check(lc, "transform_packed f0");
    }
    if (!e && tp.syn.modify)
      e = modify_run(lc, tp.syn.mod, a, m, p.f_len.data() + a, 0, (int)row, f0, sp, offs.data() + m + 1);
    if (!e && cv) {   // the slice's curve frames, read at fo[a]
      const long long d = fo[a] - fo[u0];
      ModifyCurves sc;
      sc.f0 = cv->f0 ? cv->f0 + d : nullptr; sc.ratio = cv->ratio ? cv->ratio + d : nullptr;
      e = curves_run(lc, sc, m, p.f_len.data() + a, 0, offs.data() + m + 1, p.ct.fft_size.data() + a, r.fs, (int)row,
                     f0, sp);
    }
    return lane_error(h, L, e);
  };
  auto synthesise = [&](const LaneScope &lanes, int s) {
    const int a = bounds[s], m = bounds[s + 1] - a;
    WorldB200 *L = lanes.lane(s);
    const Rows w = rows_of(a, a + m);
    unsigned char *buf = lanes.buffer(s);
    const int e = synthesis_run(&L->c, tp.syn, a, m, {(const double *)(buf + w.pf), (const double *)(buf + w.sp),
                                                      (const double *)(buf + w.ap),
                                                      (unsigned char *)y + (size_t)(yo[a] - yo[u0]) * out_bytes});
    return lane_error(h, L, e);
  };
  return transform_slices(h, bounds, bytes, analyse, synthesise);
}

// Utterances [u0, u0 + n) of a checked call: x and y point at utterance u0's rows (DEVICE; packed: its first samples);
// the request's x_lengths and per-utterance options are the call's whole arrays.  The utterances are cut into slices
// that alternate between the two lanes of a LaneScope (transform_slices).  A slice's rows (float64 input, time axis, f0,
// spectrogram, aperiodicity) live from its analysis to its synthesis in one buffer per lane, taken from the lane's pool
// and sized for its largest slice; slices are sized so that the buffer takes at most about half the lane's scratch
// budget, leaving the rest to the stages.
int transform_run(WorldB200 *h, const ChainRequest &r, const TransformPlan &tp, const void *x, int u0, int n, void *y,
                  const ModifyCurves *cv) {
  if (n <= 0) return 0;
  if (r.packed) return transform_packed_run(h, r, tp, x, u0, n, y, cv);
  const ChainPlan &p = tp.chain;
  const int f0_stride = p.f0_stride, x_stride = r.x_stride, nbit = r.nbit, row = (int)p.sp_row;
  const size_t in_row = (size_t)x_stride * (nbit ? nbit / 8 : 8);
  const size_t out_row = (size_t)tp.syn.y_stride * (tp.syn.nbit ? 2 : 8);
  struct Rows {
    size_t x, t, f, sp, ap, total;
    Rows(int m, int nbit, int x_stride, int f0_stride, int bins) {
      ArenaPlan a;
      x = a.add(nbit ? (size_t)m * x_stride * 8 : 0);
      t = a.add((size_t)m * f0_stride * 8); f = a.add((size_t)m * f0_stride * 8);
      sp = a.add((size_t)m * f0_stride * bins * 8); ap = a.add((size_t)m * f0_stride * bins * 8);
      total = a.total;
    }
  };
  auto rows_of = [&](int m) { return Rows(m, nbit, x_stride, f0_stride, row); };
  int n_slices = 1;
  {
#ifndef WB_EMU
    const bool two = n > 1;
#else
    const bool two = false;
#endif
    const double lane_budget = (double)h->c.scratch_budget / (two ? 2.0 : 1.0);
    const int fit = (int)dmax(1.0, dmin((double)n, lane_budget / 2.0 / (double)rows_of(1).total));
    n_slices = (n + fit - 1) / fit;
    if (two) n_slices = imin(n, (n_slices + 1) / 2 * 2);   // an even count: both lanes get the same work
  }
  std::vector<int> bounds(n_slices + 1);
  for (int s = 0; s <= n_slices; ++s) bounds[s] = (int)((long long)n * s / n_slices);
  // slice s: its lane, the global index of its first utterance, its size and where its rows are
  auto slice = [&](const LaneScope &lanes, int s, WorldB200 **L, int *g, int *m, double **xs, double **t, double **f,
                   double **sp, double **ap) {
    const Rows at = rows_of(lanes.most(s));
    unsigned char *rows = lanes.buffer(s);
    *L = lanes.lane(s); *g = u0 + bounds[s]; *m = bounds[s + 1] - bounds[s];
    *xs = (double *)(rows + at.x); *t = (double *)(rows + at.t); *f = (double *)(rows + at.f);
    *sp = (double *)(rows + at.sp); *ap = (double *)(rows + at.ap);
  };
  auto analyse = [&](const LaneScope &lanes, int s) {
    WorldB200 *L; int g, m; double *xd, *t, *f, *sp, *ap;
    slice(lanes, s, &L, &g, &m, &xd, &t, &f, &sp, &ap);
    const unsigned char *xin = (const unsigned char *)x + (size_t)bounds[s] * in_row;
    const double *xs = nbit ? xd : (const double *)xin;
    int e = nbit ? world_b200_pcm_to_double_batch(L, xin, nbit, m, x_stride, r.x_lengths ? r.x_lengths + g : nullptr, xd)
                 : 0;
    if (!e) e = dev_memset(&L->c, t, 0, (size_t)m * f0_stride * 8);
    if (!e) e = dev_memset(&L->c, f, 0, (size_t)m * f0_stride * 8);
    if (!e) e = chain_f0(L, r, p, g, m, xs, t, f);
    if (!e) e = chain_spectral(L, r, p, g, m, xs, t, f, sp, ap);
    if (!e && tp.syn.modify) e = modify_run(&L->c, tp.syn.mod, g, m, p.f_len.data() + g, f0_stride, row, f, sp);
    return lane_error(h, L, e);
  };
  auto synthesise = [&](const LaneScope &lanes, int s) {
    WorldB200 *L; int g, m; double *xd, *t, *f, *sp, *ap;
    slice(lanes, s, &L, &g, &m, &xd, &t, &f, &sp, &ap);
    const int e = synthesis_run(&L->c, tp.syn, g, m, {f, sp, ap, (unsigned char *)y + (size_t)bounds[s] * out_row});
    return lane_error(h, L, e);
  };
  return transform_slices(h, bounds, [&](int s) { return rows_of(bounds[s + 1] - bounds[s]).total; }, analyse,
                          synthesise);
}

}  // namespace wb

extern "C" {

int world_b200_transform_samples(int fs, int x_length, double frame_period, double time_scale) {
  const double fp = frame_period * time_scale;
  if (!(fp > 0.0) || !isfinite(fp)) return 0;
  const double v = (frames_for(fs, x_length, frame_period) - 1) * fp / 1000.0 * fs;
  return v < 2147483646.0 ? static_cast<int>(v) + 1 : 0;
}

int world_b200_transform_batch(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths,
                               int fs, const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                               const DioOption *dio_options, const double *f0_scale, const double *spectral_ratio,
                               const double *time_scale, int nbit_out, void *y, int y_stride, int *y_lengths) {
  return world_b200_transform_batch_spectral_options(h, x, nbit, n_utts, x_stride, x_lengths, fs, option,
                                                     harvest_options, dio_options, nullptr, nullptr, f0_scale,
                                                     spectral_ratio, time_scale, nbit_out, y, y_stride, y_lengths);
}

int world_b200_transform_batch_spectral_options(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride,
                                                const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                                const HarvestOption *harvest_options, const DioOption *dio_options,
                                                const CheapTrickOption *cheaptrick_options,
                                                const D4COption *d4c_options, const double *f0_scale,
                                                const double *spectral_ratio, const double *time_scale, int nbit_out,
                                                void *y, int y_stride, int *y_lengths) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  ChainRequest r(x, nbit, n_utts, x_stride, x_lengths, fs, option, nullptr, nullptr, 0, nullptr, nullptr);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options;
  r.transform = true;
  TransformPlan tp;
  const int rc = transform_check(h, r, f0_scale, spectral_ratio, time_scale, nbit_out, y, y_stride, "transform_batch", &tp);
  if (rc) return rc;
  if (y_lengths) std::copy(tp.syn.y_len.begin(), tp.syn.y_len.end(), y_lengths);
  return transform_run(h, r, tp, x, 0, n_utts, y);
}

int world_b200_transform_packed_samples(int fs, int n_utts, const long long *x_offsets, double frame_period,
                                        const double *time_scale, long long *y_offsets) {
  if (fs <= 0 || n_utts < 0 || !(frame_period > 0.0) || !y_offsets) return WORLD_B200_EINVAL;
  std::vector<int> x_len;
  std::vector<long long> f_off;
  if (!packed_layout(fs, n_utts, x_offsets, frame_period, &x_len, &f_off).empty()) return WORLD_B200_EINVAL;
  std::vector<long long> y_off(1, 0);
  for (int u = 0; u < n_utts; ++u) {
    const double ts = time_scale ? time_scale[u] : 1.0;
    const int y_len = world_b200_transform_samples(fs, x_len[u], frame_period, ts);
    if (!(ts > 0.0) || !isfinite(ts) || y_len == 0) return WORLD_B200_EINVAL;
    y_off.push_back(y_off.back() + y_len);
  }
  std::copy(y_off.begin(), y_off.end(), y_offsets);
  return 0;
}

}  // extern "C"

// world_b200_transform_packed, and with cv (factors null) world_b200_transform_packed_curves: the curves are checked
// on the device after every host check, before any work is queued
static int transform_packed(WorldB200 *h, const void *x, int nbit, int n_utts, const long long *x_offsets, int fs,
                            const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                            const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                            const D4COption *d4c_options, const double *f0_scale, const double *spectral_ratio,
                            const double *time_scale, int nbit_out, void *y, long long *y_offsets,
                            const ModifyCurves *cv) {
  if (!h) return WORLD_B200_EINVAL;
  if (n_utts == 0) {   // as the packed synthesis calls: nothing to check against, nothing to queue
    if (y_offsets) y_offsets[0] = 0;
    return 0;
  }
  DeviceGuard guard_(&h->c);
  ChainRequest r = packed_request(x, nbit, n_utts, x_offsets, fs, option, harvest_options, dio_options,
                                  cheaptrick_options, d4c_options, nullptr, nullptr, nullptr, nullptr);
  r.transform = true;
  TransformPlan tp;
  const char *who = cv ? "transform_packed_curves" : "transform_packed";
  int rc = transform_check(h, r, f0_scale, spectral_ratio, time_scale, nbit_out, y, 0, who, &tp);
  const ChainPlan &p = tp.chain;
  if (!rc && cv) rc = curves_check(&h->c, who, *cv, n_utts, p.f_len.data(), 0, p.f_off.data(), p.ct.fft_size.data());
  if (rc) return rc;
  if (y_offsets) std::copy(tp.syn.y_off.begin(), tp.syn.y_off.end(), y_offsets);
  return transform_run(h, r, tp, x, 0, n_utts, y, cv);
}

extern "C" {

int world_b200_transform_packed(WorldB200 *h, const void *x, int nbit, int n_utts, const long long *x_offsets, int fs,
                                const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                                const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                                const D4COption *d4c_options, const double *f0_scale, const double *spectral_ratio,
                                const double *time_scale, int nbit_out, void *y, long long *y_offsets) {
  return transform_packed(h, x, nbit, n_utts, x_offsets, fs, option, harvest_options, dio_options, cheaptrick_options,
                          d4c_options, f0_scale, spectral_ratio, time_scale, nbit_out, y, y_offsets, nullptr);
}

int world_b200_transform_packed_curves(WorldB200 *h, const void *x, int nbit, int n_utts, const long long *x_offsets,
                                       int fs, const WorldB200AnalysisOption *option,
                                       const HarvestOption *harvest_options, const DioOption *dio_options,
                                       const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                       const double *f0_curve, const double *spectral_ratio_curve,
                                       const double *time_scale, int nbit_out, void *y, long long *y_offsets) {
  ModifyCurves cv;
  cv.f0 = f0_curve; cv.ratio = spectral_ratio_curve;
  return transform_packed(h, x, nbit, n_utts, x_offsets, fs, option, harvest_options, dio_options, cheaptrick_options,
                          d4c_options, nullptr, nullptr, time_scale, nbit_out, y, y_offsets, &cv);
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
  return analyze_chain(h, ChainRequest(x, 0, n, x_stride, x_lengths, fs, opt, time_axis_full, f0_full, f0_stride,
                                       spectrogram_full, aperiodicity_full), true);
}

int world_b200_analyze_batch_allgather_options(WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths,
                                               int fs, const WorldB200AnalysisOption *opt,
                                               const HarvestOption *harvest_options, double *time_axis_full,
                                               double *f0_full, int f0_stride, double *spectrogram_full,
                                               double *aperiodicity_full) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  ChainRequest r(x, 0, n, x_stride, x_lengths, fs, opt, time_axis_full, f0_full, f0_stride, spectrogram_full,
                 aperiodicity_full);
  r.harvest_options = harvest_options;
  return analyze_chain(h, r, true);
}

int world_b200_analyze_batch_allgather_dio_options(WorldB200 *h, const double *x, int n, int x_stride,
                                                   const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                   const DioOption *dio_options, double *time_axis_full,
                                                   double *f0_full, int f0_stride, double *spectrogram_full,
                                                   double *aperiodicity_full) {
  if (!dio_options) return WORLD_B200_EINVAL;
  ChainRequest r(x, 0, n, x_stride, x_lengths, fs, opt, time_axis_full, f0_full, f0_stride, spectrogram_full,
                 aperiodicity_full);
  r.dio_options = dio_options;
  return analyze_chain(h, r, true);
}

int world_b200_analyze_batch_allgather_spectral_options(
    WorldB200 *h, const double *x, int n, int x_stride, const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
    const HarvestOption *harvest_options, const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
    const D4COption *d4c_options, double *time_axis_full, double *f0_full, int f0_stride, int row_stride,
    double *spectrogram_full, double *aperiodicity_full) {
  ChainRequest r(x, 0, n, x_stride, x_lengths, fs, opt, time_axis_full, f0_full, f0_stride, spectrogram_full,
                 aperiodicity_full);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options; r.row_stride = row_stride;
  return analyze_chain(h, r, true);
}

// The device chain with coded rows out (and PCM or doubles in): analyze_chain with the fused coded frame kernels.
int world_b200_analyze_coded_batch(WorldB200 *h, const void *x, int nbit, int n, int x_stride, const int *x_lengths,
                                   int fs, const WorldB200AnalysisOption *opt, int number_of_dimensions,
                                   double *time_axis, double *f0, int f0_stride, double *coded_spectral_envelope,
                                   double *coded_aperiodicity) {
  return analyze_chain(h, coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                        f0_stride, coded_spectral_envelope, coded_aperiodicity), false);
}

int world_b200_analyze_coded_batch_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                           const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                           const HarvestOption *harvest_options, int number_of_dimensions,
                                           double *time_axis, double *f0, int f0_stride,
                                           double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  ChainRequest r = coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                 f0_stride, coded_spectral_envelope, coded_aperiodicity);
  r.harvest_options = harvest_options;
  return analyze_chain(h, r, false);
}

int world_b200_analyze_coded_batch_dio_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                               const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                               const DioOption *dio_options, int number_of_dimensions,
                                               double *time_axis, double *f0, int f0_stride,
                                               double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  ChainRequest r = coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                 f0_stride, coded_spectral_envelope, coded_aperiodicity);
  r.dio_options = dio_options;
  return analyze_chain(h, r, false);
}

int world_b200_analyze_coded_batch_spectral_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                                    const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                    const HarvestOption *harvest_options, const DioOption *dio_options,
                                                    const CheapTrickOption *cheaptrick_options,
                                                    const D4COption *d4c_options, int number_of_dimensions,
                                                    double *time_axis, double *f0, int f0_stride,
                                                    double *coded_spectral_envelope, double *coded_aperiodicity) {
  ChainRequest r = coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                 f0_stride, coded_spectral_envelope, coded_aperiodicity);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options;
  return analyze_chain(h, r, false);
}

// The packed chains on device arrays: one plan, then packed_run over every utterance.  f_offsets (HOST, may be NULL)
// receives the plan's frame offsets once the request is checked.
static int analyze_packed_chain(WorldB200 *h, const ChainRequest &r, long long *f_offsets) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  const char *who = r.coded ? "analyze_coded_packed" : "analyze_packed";
  if (r.n > 0 && (!r.time_axis || !r.f0)) {
    h->c.last_error = std::string(who) + ": time_axis and f0 must be given";
    return WORLD_B200_EINVAL;
  }
  ChainPlan p;
  int rc = chain_plan(&h->c, r, who, &p);
  if (rc) return rc;
  if (f_offsets) std::copy(p.f_off.begin(), p.f_off.end(), f_offsets);
  if (r.n == 0) return 0;
  return packed_run(h, r, p, 0, r.n, r.x, r.time_axis, r.f0, p.want_sp ? r.spectrogram : nullptr,
                    p.want_ap ? r.aperiodicity : nullptr);
}

int world_b200_packed_frames(int fs, int n, const long long *x_offsets, double frame_period, long long *f_offsets) {
  if (fs <= 0 || n < 0 || !(frame_period > 0.0) || !f_offsets) return WORLD_B200_EINVAL;
  std::vector<int> x_len;
  std::vector<long long> f_off;
  if (!packed_layout(fs, n, x_offsets, frame_period, &x_len, &f_off).empty()) return WORLD_B200_EINVAL;
  std::copy(f_off.begin(), f_off.end(), f_offsets);
  return 0;
}

int world_b200_analyze_packed(WorldB200 *h, const double *x, int n, const long long *x_offsets, int fs,
                              const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                              const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                              const D4COption *d4c_options, double *time_axis, double *f0, int row_stride,
                              double *spectrogram, double *aperiodicity, long long *f_offsets) {
  ChainRequest r = packed_request(x, 0, n, x_offsets, fs, opt, harvest_options, dio_options, cheaptrick_options,
                                  d4c_options, time_axis, f0, spectrogram, aperiodicity);
  r.row_stride = row_stride;
  return analyze_packed_chain(h, r, f_offsets);
}

int world_b200_analyze_coded_packed(WorldB200 *h, const void *x, int nbit, int n, const long long *x_offsets, int fs,
                                    const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                    const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                                    const D4COption *d4c_options, int number_of_dimensions, double *time_axis,
                                    double *f0, double *coded_spectral_envelope, double *coded_aperiodicity,
                                    long long *f_offsets) {
  ChainRequest r = packed_request(x, nbit, n, x_offsets, fs, opt, harvest_options, dio_options, cheaptrick_options,
                                  d4c_options, time_axis, f0, coded_spectral_envelope, coded_aperiodicity);
  r.coded = true; r.dims = number_of_dimensions;
  return analyze_packed_chain(h, r, f_offsets);
}

int world_b200_analyze_coded_batch_allgather(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                             const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                             int number_of_dimensions, double *time_axis_full, double *f0_full,
                                             int f0_stride, double *coded_spectral_envelope_full,
                                             double *coded_aperiodicity_full) {
  return analyze_chain(h, coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis_full,
                                        f0_full, f0_stride, coded_spectral_envelope_full, coded_aperiodicity_full), true);
}

int world_b200_analyze_coded_batch_allgather_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                                     const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                     const HarvestOption *harvest_options, int number_of_dimensions,
                                                     double *time_axis_full, double *f0_full, int f0_stride,
                                                     double *coded_spectral_envelope_full,
                                                     double *coded_aperiodicity_full) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  ChainRequest r = coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis_full,
                                 f0_full, f0_stride, coded_spectral_envelope_full, coded_aperiodicity_full);
  r.harvest_options = harvest_options;
  return analyze_chain(h, r, true);
}

int world_b200_analyze_coded_batch_allgather_dio_options(WorldB200 *h, const void *x, int nbit, int n, int x_stride,
                                                         const int *x_lengths, int fs,
                                                         const WorldB200AnalysisOption *opt,
                                                         const DioOption *dio_options, int number_of_dimensions,
                                                         double *time_axis_full, double *f0_full, int f0_stride,
                                                         double *coded_spectral_envelope_full,
                                                         double *coded_aperiodicity_full) {
  if (!dio_options) return WORLD_B200_EINVAL;
  ChainRequest r = coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis_full,
                                 f0_full, f0_stride, coded_spectral_envelope_full, coded_aperiodicity_full);
  r.dio_options = dio_options;
  return analyze_chain(h, r, true);
}

int world_b200_analyze_coded_batch_allgather_spectral_options(
    WorldB200 *h, const void *x, int nbit, int n, int x_stride, const int *x_lengths, int fs,
    const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options, const DioOption *dio_options,
    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options, int number_of_dimensions,
    double *time_axis_full, double *f0_full, int f0_stride, double *coded_spectral_envelope_full,
    double *coded_aperiodicity_full) {
  ChainRequest r = coded_request(x, nbit, n, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis_full,
                                 f0_full, f0_stride, coded_spectral_envelope_full, coded_aperiodicity_full);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options;
  return analyze_chain(h, r, true);
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
  rng_fill(ctx, out_dev, (unsigned)first, (unsigned)(first + n));
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
