// wb_rng.cu -- exact, parallel reproduction of the reference's sequential randn() stream.
//
// Reference: matlabfunctions.cpp:237-264 (xorshift128 seeded (123456789, 362436069, 521288629,
// 88675123); one randn() = 12 state steps, value = sum(w >> 4) / 2^28 - 6), reseeded once per
// CheapTrick()/D4C() call (cheaptrick.cpp:205-206, d4c.cpp:345-346) and consumed frame after
// frame, so frame i's noise depends on how many draws frames 0..i-1 took.
//
// GPU restatement: the draw counts per frame are a pure function of f0 (counted by the
// stage's own kernel), an exclusive scan gives every frame its offset into the utterance's
// stream, and the stream itself -- the same for every utterance -- is materialised once per
// context (rng_table_reserve) by `rng_fill_kernel`: thread g produces draws
// [128 g, 128 g + 128) after jumping there with popcount(g) GF(2) matrix-vector products
// (xorshift128 is linear over GF(2); J_k = T^(12*128*2^k) are precomputed on the host as
// 4-bit lookup tables).  Draws are stored as the exact uint32 sum so consumers evaluate
// `sum / 268435456.0 - 6.0` in FP64 exactly like the reference.
#include "wb_internal.h"

namespace wb {

// ------------------------------------------------------------------ host: jump tables
namespace {
struct U128 { uint32_t v[4]; };
inline U128 xs_step(U128 s) {
  uint32_t t = s.v[0] ^ (s.v[0] << 11);
  U128 r;
  r.v[0] = s.v[1]; r.v[1] = s.v[2]; r.v[2] = s.v[3];
  r.v[3] = (s.v[3] ^ (s.v[3] >> 19)) ^ (t ^ (t >> 8));
  return r;
}
inline U128 x128(U128 a, const U128 &b) {
  for (int i = 0; i < 4; ++i) a.v[i] ^= b.v[i];
  return a;
}
struct BitMat { U128 col[128]; };
inline U128 matvec(const BitMat &m, const U128 &x) {
  U128 r = {{0, 0, 0, 0}};
  for (int b = 0; b < 128; ++b)
    if ((x.v[b >> 5] >> (b & 31)) & 1u) r = x128(r, m.col[b]);
  return r;
}
}  // namespace

void rng_build_jump_tables(uint32_t *tables /* [WB_RNG_NJ][32][16][4] */) {
  BitMat *j = new BitMat;
  for (int b = 0; b < 128; ++b) {
    U128 e = {{0, 0, 0, 0}};
    e.v[b >> 5] = 1u << (b & 31);
    for (int s = 0; s < 12 * WB_RNG_CHUNK; ++s) e = xs_step(e);
    j->col[b] = e;
  }
  BitMat *sq = new BitMat;
  for (int k = 0; k < WB_RNG_NJ; ++k) {
    for (int p = 0; p < 32; ++p)
      for (int v = 0; v < 16; ++v) {
        U128 r = {{0, 0, 0, 0}};
        for (int b = 0; b < 4; ++b)
          if ((v >> b) & 1) r = x128(r, j->col[4 * p + b]);
        uint32_t *dst = tables + ((size_t)(k * 32 + p) * 16 + v) * 4;
        for (int i = 0; i < 4; ++i) dst[i] = r.v[i];
      }
    for (int b = 0; b < 128; ++b) sq->col[b] = matvec(*j, j->col[b]);
    *j = *sq;
  }
  delete j;
  delete sq;
}

// ------------------------------------------------------------------ device
WB_DEV uint4 rng_apply(const uint4 *__restrict__ tab /* [32][16] */, uint4 s) {
  uint4 r = make_uint4(0u, 0u, 0u, 0u);
  const unsigned w[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const unsigned nib = (w[p >> 3] >> (4 * (p & 7))) & 15u;
    const uint4 t = __ldg(&tab[p * 16 + nib]);
    r.x ^= t.x; r.y ^= t.y; r.z ^= t.z; r.w ^= t.w;
  }
  return r;
}

WB_DEV unsigned rng_draw(uint4 &s) {
  unsigned acc = 0;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const unsigned t = s.x ^ (s.x << 11);
    s.x = s.y; s.y = s.z; s.z = s.w;
    s.w = (s.w ^ (s.w >> 19)) ^ (t ^ (t >> 8));
    acc += s.w >> 4;
  }
  return acc;
}

// grid: ceil(chunks / 32 / WB_RNG_WARPS); block: 32*WB_RNG_WARPS threads; each warp produces 32 chunks of
// WB_RNG_CHUNK draws = 4096 consecutive draws, stored coalesced via a smem tile.  Draws [first, total) of the stream,
// draw d at dst[d - first]; the context's table takes first = 0, the window hook any first.  total is at most
// WB_RNG_REACH, so chunk g < 2^WB_RNG_NJ and no draw index wraps.
WB_KERNEL_PLAIN rng_fill_kernel(const uint4 *__restrict__ jump, unsigned *__restrict__ dst, unsigned first,
                                unsigned total) {
  const unsigned chunk0 = first / WB_RNG_CHUNK;
  // draw d goes to dst[d - first] if d - first < span: one unsigned compare (d < first wraps past span)
  const unsigned span = total > first ? total - first : 0u;
#ifdef WB_EMU
  // flat emulation: one "thread" = one chunk
  const unsigned g = chunk0 + blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned start = g * WB_RNG_CHUNK;
  if (start >= total) return;
  uint4 s = make_uint4(123456789u, 362436069u, 521288629u, 88675123u);
  for (int k = 0; k < WB_RNG_NJ; ++k)
    if ((g >> k) & 1u) s = rng_apply(jump + (size_t)k * 512, s);
  for (unsigned i = 0; i < WB_RNG_CHUNK && start + i < total; ++i) {
    const unsigned v = rng_draw(s), rel = start + i - first;
    if (rel < span) dst[rel] = v;
  }
#else
  __shared__ unsigned tile[WB_RNG_WARPS][32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned g = chunk0 + (blockIdx.x * WB_RNG_WARPS + warp) * 32 + lane;
  const unsigned warp_first = (chunk0 + (blockIdx.x * WB_RNG_WARPS + warp) * 32) * WB_RNG_CHUNK;
  if (warp_first >= total) return;  // whole warp leaves together
  const unsigned warp_rel = warp_first - first;
  uint4 s = make_uint4(123456789u, 362436069u, 521288629u, 88675123u);
  if (g * WB_RNG_CHUNK < total)
    for (int k = 0; k < WB_RNG_NJ; ++k)
      if ((g >> k) & 1u) s = rng_apply(jump + (size_t)k * 512, s);
  for (int c = 0; c < WB_RNG_CHUNK / 32; ++c) {
#pragma unroll 4
    for (int i = 0; i < 32; ++i) tile[warp][lane][i] = rng_draw(s);
    __syncwarp();
    for (int row = 0; row < 32; ++row) {
      const unsigned rel = warp_rel + row * WB_RNG_CHUNK + c * 32 + lane;
      if (rel < span) dst[rel] = tile[warp][row][lane];
    }
    __syncwarp();
  }
#endif
}

void rng_fill(const Ctx *ctx, unsigned *out, unsigned first, unsigned end) {
  if (end <= first) return;
  const size_t chunk0 = first / WB_RNG_CHUNK;
  const size_t chunks = ((size_t)end + WB_RNG_CHUNK - 1) / WB_RNG_CHUNK - chunk0;
  const unsigned per_block = 32 * WB_RNG_WARPS;
  WB_LAUNCH_FLAT(rng_fill_kernel, dim3((unsigned)((chunks + per_block - 1) / per_block)), per_block, 0, ctx->stream,
                 reinterpret_cast<const uint4 *>(ctx->rng_jump), out, first, end);
}

// ------------------------------------------------------------------ the context's stream table
// Every utterance of every call reads the same stream from draw 0 (the reference reseeds at each call), so one table
// serves them all; a frame's draws are table + its offset.  The table is sized to the largest per-utterance bound a call
// asked for, plus an eighth, in steps of 2^20 draws (4 MB): calls of similar shapes do not grow it again.  A context
// starts with one step (ctx_init_tables), so calls on short utterances never grow it.
const unsigned *rng_table_reserve(Ctx *ctx, size_t draws) {
  if (ctx->rng_table && draws <= ctx->rng_table_len) return ctx->rng_table;
  const size_t step = (size_t)1 << 20;
  const size_t len = (draws + draws / 8 + step - 1) / step * step;
  // kernels queued on the stream may still read the old table
  if (ctx->rng_table) {
    if (dev_sync(ctx)) return nullptr;
    dev_free(ctx->rng_table);
    ctx->rng_table = nullptr;
    ctx->rng_table_len = 0;
  }
  unsigned *t = (unsigned *)dev_malloc(ctx, len * sizeof(unsigned));
  if (!t) return nullptr;
  rng_fill(ctx, t, 0, (unsigned)(len < WB_RNG_REACH ? len : WB_RNG_REACH));
  if (dev_check(ctx, "randn table")) { dev_free(t); return nullptr; }
  ctx->rng_table = t;
  ctx->rng_table_len = len;
  return t;
}

// ------------------------------------------------------------------ per-utterance scans
// counts[u][0..len_u) -> exclusive offsets (same layout) + totals[u] (+ base[u] added to every
// offset, used by D4C's second pass which continues the stream after the first pass).  The sums
// run in 64 bits: a total beyond WB_RNG_REACH sets status bit 8 (world_b200_synchronize reports
// WORLD_B200_EDOMAIN) and is stored clamped to the reach.
// utt_off: utterance u's counts and offsets start at utt_off[u] (packed; null: at u * stride).
WB_KERNEL_PLAIN scan_counts_kernel(const unsigned *__restrict__ counts, const int *__restrict__ lens,
                                   int stride, const unsigned *__restrict__ base,
                                   unsigned *__restrict__ offsets, unsigned *__restrict__ totals,
                                   int *__restrict__ status, const long long *__restrict__ utt_off) {
  WB_SHARED unsigned long long part[1025];
  const int utt = blockIdx.x, tid = WB_TID, nth = WB_NTH;
  const int len = lens[utt];
  const size_t at = utt_off ? (size_t)utt_off[utt] : (size_t)utt * stride;
  const unsigned *c = counts + at;
  unsigned *o = offsets + at;
  const int chunk = (len + nth - 1) / nth;
  const int lo = imin(len, tid * chunk), hi = imin(len, lo + chunk);
  unsigned long long s = 0;
  for (int i = lo; i < hi; ++i) s += c[i];
  part[tid] = s;
  WB_SYNC();
  if (tid == 0) {
    unsigned long long run = base ? base[utt] : 0u;
    for (int t = 0; t < nth; ++t) { const unsigned long long v = part[t]; part[t] = run; run += v; }
    if (run > WB_RNG_REACH) {
      atomicOr_status(status, 8);
      run = WB_RNG_REACH;
    }
    totals[utt] = (unsigned)run;
  }
  WB_SYNC();
  unsigned long long run = part[tid];
  for (int i = lo; i < hi; ++i) { const unsigned v = c[i]; o[i] = (unsigned)run; run += v; }
}

void scan_counts(const Ctx *ctx, const unsigned *counts, const int *lens_dev, int stride,
                 const unsigned *base, unsigned *offsets, unsigned *totals, int n_utts,
                 const long long *utt_off) {
  if (n_utts <= 0) return;
  WB_LAUNCH_COOP(scan_counts_kernel, dim3((unsigned)n_utts), 256, 0, ctx->stream, counts, lens_dev,
                 stride, base, offsets, totals, ctx->status_dev, utt_off);
}

}  // namespace wb
