// wb_cheaptrick.cu -- K-CT: spectral envelope, one CTA per (utterance, frame).
//
// Replaces the frame loop of CheapTrick() (cheaptrick.cpp:200-229) and its helpers
// (GetWindowedWaveform :112-142, GetPowerSpectrum :64-82, AddInfinitesimalNoise :147-151,
// SmoothingWithRecovery :22-57) plus common.cpp's DCCorrection/LinearSmoothing.  Algorithm card:
// SURVEY.md A1.  Everything between the waveform read and the spectrogram row write stays in
// shared memory: three real FFTs (window spectrum, cepstrum, liftered cepstrum back -- the
// last two are transforms of real even sequences, so the reference's c2r is a forward r2c
// here), the index-order running sum of LinearSmoothing on one thread, log/exp fused in.
//
// HBM traffic per frame (algorithmic): (2h+1)*8 B of waveform (L2 hits after the first frame of
// a hop), 16 B of f0/time, (2h+1 + fft/2+1)*4 B of materialised draws, (fft/2+1)*8 B written.
#include "wb_internal.h"
#include "wb_spectral.cuh"
#include <stdlib.h>

namespace wb {

struct CtParams {
  const double *x; const int *x_len; int x_stride;
  const double *time_axis; const double *f0; const int *f_len; int f_stride;
  int fs, fft_size, lg_fft;
  double q1, f0_floor;
  const unsigned *draws;  // the context's stream table: a frame's draws start at its draw_off entry
  const unsigned *draw_off;
  double *out;            // [n][f_stride][out_stride], or (f_off) [F][out_stride]
  int out_stride;         // doubles per spectrogram row (fft/2+1 unless the caller pads its rows)
  const int *uid;         // [n] batch index of the launch's utterance blockIdx.y; null: blockIdx.y itself
  const long long *f_off; // [n] packed rows: output frame of each utterance's frame 0; null: u * f_stride
  // packed inputs: utterance u's samples at x + x_off[u], its frames (time_axis, f0 and output) at f_off[u] + i, and
  // the launch's utterance ul's draw offsets at cum[ul] + i (cum: [n + 1] frames of the launch's utterances before
  // it); null: padded inputs
  const long long *x_off, *cum;
  int n_launch;           // packed: utterances of the launch (entries of cum)
  const double2 *tw;
  int *status;
  // coded tail (ct_coded_kernel): mel interpolation + DCT of the log envelope, CodeSpectralEnvelope (codec.cpp:279-295)
  int c_dims; const int *c_idx; const double *c_frac; const double2 *c_weight; double c_norm;
  double *c_out;          // [n][f_stride][c_dims], or (f_off) [F][c_dims]
};

WB_DEV double ct_effective_f0(double f0, double f0_floor) {
  return f0 <= f0_floor ? 500.0 : f0;  // kDefaultF0, cheaptrick.cpp:218
}

// draws consumed by frame = window samples + spectrum bins (SURVEY.md A1)
WB_KERNEL_PLAIN ct_count_kernel(const double *__restrict__ f0, const int *__restrict__ f_len,
                                int f_stride, int n_utts, int fs, int fft_size, double f0_floor,
                                const int *__restrict__ uid, unsigned *__restrict__ counts) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_utts * f_stride) return;
  const int ul = (int)(g / f_stride), i = (int)(g % f_stride);   // f_len and counts follow the launch's order
  unsigned c = 0;
  if (i < f_len[ul]) {
    const size_t fidx = uid ? (size_t)uid[ul] * f_stride + i : (size_t)g;
    const double f = ct_effective_f0(f0[fidx], f0_floor);
    const int h = round_half_away(1.5 * fs / f);
    c = (unsigned)(2 * h + 1) + (unsigned)(fft_size / 2 + 1);
  }
  counts[g] = c;
}

// the same over packed inputs: one thread per frame of the launch's utterances, frame g of utterance ul at cum[ul] + i
WB_KERNEL_PLAIN ct_count_packed_kernel(const double *__restrict__ f0, const long long *__restrict__ f_off,
                                       const long long *__restrict__ cum, int n_utts, int fs, int fft_size,
                                       double f0_floor, const int *__restrict__ uid, unsigned *__restrict__ counts) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= cum[n_utts]) return;
  const int ul = packed_find(cum, n_utts, g);
  const int u = uid ? uid[ul] : ul;
  const double f = ct_effective_f0(f0[f_off[u] + (g - cum[ul])], f0_floor);
  const int h = round_half_away(1.5 * fs / f);
  counts[g] = (unsigned)(2 * h + 1) + (unsigned)(fft_size / 2 + 1);
}

// Shared memory: two padded complex buffers of fft_size/2 slots (the FFT ping-pongs between them, wb_fft.cuh)
// + the reduction scratch.  Between transforms the buffer that does not hold FFT input serves as the plain
// double array of the phase (window, power spectrum, smoothing scratch), so nothing else is needed.
WB_HD inline size_t ct_smem_bytes(int fft_size) {
  return (size_t)2 * WB_FPAD_SLOTS(fft_size / 2) * sizeof(double2) + WB_RED_DOUBLES * sizeof(double);
}

// kPacked: packed inputs (p.x_off, p.cum), a compile-time choice so that the padded kernels keep their own code
template <bool kCoded, bool kPacked>
WB_DEV void ct_frame_body(const CtParams &p) {
  WB_DYN_SMEM(double2, smem2);
  const int tid = WB_TID, nth = WB_NTH;
  // f_len and draw offsets follow the launch's order.  Packed: the grid runs over the launch's packed frames (none of it
  // idles on short utterances), blockIdx.x being frame i of launch entry ul, its draw offsets' index
  int ul, i;
  if (kPacked) {
    ul = packed_find(p.cum, p.n_launch, (long long)blockIdx.x);
    i = (int)((long long)blockIdx.x - p.cum[ul]);
  } else {
    ul = blockIdx.y;
    i = blockIdx.x;
    if (i >= p.f_len[ul]) return;
  }
  const int u = p.uid ? __ldg(p.uid + ul) : ul;
  const int N = p.fft_size, half = N / 2;
  const int slots = WB_FPAD_SLOTS(half);
  double2 *A = smem2, *B = smem2 + slots;
  double *red = reinterpret_cast<double *>(B + slots);   // WB_RED_DOUBLES

  // only the addresses differ between the padded and the packed layouts: the output row, and with packed inputs the
  // input frame, the samples and the draw offset
  const size_t fidx = kPacked ? (size_t)(p.f_off[u] + i) : (size_t)u * p.f_stride + i;
  const size_t oidx = p.f_off ? (size_t)(p.f_off[u] + i) : fidx;
  const double f = ct_effective_f0(p.f0[fidx], p.f0_floor);
  const double t = p.time_axis[fidx];
  const int fs = p.fs;
  const int x_len = p.x_len[u];
  const double *x = kPacked ? p.x + p.x_off[u] : p.x + (size_t)u * p.x_stride;
  const unsigned *draw = p.draws + p.draw_off[kPacked ? (size_t)blockIdx.x : (size_t)ul * p.f_stride + i];

  const int h = round_half_away(1.5 * fs / f);
  const int nwin = 2 * h + 1;
  if (nwin > N) {  // f0 below the floor implied by fft_size: undefined in the reference
    if (tid == 0) atomicOr_status(p.status, 1);
    return;
  }
  const int origin = round_half_away(t * fs + 0.001);

  // ---- F0-adaptive Hanning window, normalised to unit energy (cheaptrick.cpp:97-106)
  double *za = reinterpret_cast<double *>(A);   // packed FFT input: sample e at rpad(e)
  double *wv = reinterpret_cast<double *>(B);   // window values
  double sq = 0.0;
  for (int j = tid; j < nwin; j += nth) {
    const double pos = (j - h) / 1.5 / fs;
    const double w = 0.5 * cos_small(kPi * pos * f) + 0.5;
    wv[j] = w;
    sq += w * w;
  }
  // first round's sample and draw requested before the reduction's barriers, every later round's one round ahead
  double x_next = 0.0;
  unsigned d_next = 0u;
  if (tid < nwin) { x_next = x[imin(x_len - 1, imax(0, origin + tid - h))]; d_next = draw[tid]; }
  const double norm = sqrt(block_sum(sq, red));
  // ---- windowed waveform + 1e-12 * randn, weighted-mean removal (:126-137)
  double s1 = 0.0, s2 = 0.0;
  for (int j = tid; j < nwin; j += nth) {
    const double x_now = x_next;
    const unsigned d_now = d_next;
    if (j + nth < nwin) { x_next = x[imin(x_len - 1, imax(0, origin + j + nth - h))]; d_next = draw[j + nth]; }
    const double w = wv[j] / norm;
    wv[j] = w;
    const double v = x_now * w + randn_value(d_now) * kTiny;
    za[rpad(j)] = v;
    s1 += v;
    s2 += w;
  }
  block_sum2(s1, s2, red);
  const double coef = s1 / s2;
  for (int j = tid; j < N; j += nth) za[rpad(j)] = (j < nwin) ? za[rpad(j)] - wv[j] * coef : 0.0;
  WB_SYNC();

  // ---- power spectrum (:71-78): the unpack of the real FFT squares straight into the idle buffer
  const int lgc = p.lg_fft - 1;
  double2 *z = sfft_forward(A, B, lgc, p.tw);
  double2 *o = (z == A) ? B : A;
  double *pw = reinterpret_cast<double *>(o);
  rfft_unpack(z, p.lg_fft, p.tw, [&](int k, double2 c) { pw[k] = c.x * c.x + c.y * c.y; });
  WB_SYNC();
  // the draws of the +eps noise below are requested now: they arrive while the smoothing (barriers, one thread's
  // index-order running sum) keeps the CTA waiting anyway.  (half + 1 <= 5 * 128 up to fft_size 1024; beyond that
  // the tail of the loop below loads as before.)
  unsigned dpre[5];
#pragma unroll
  for (int q = 0; q < 5; ++q) { const int k = tid + q * nth; dpre[q] = (k <= half) ? draw[nwin + k] : 0u; }
  dc_correction<true>(pw, f, fs, N, reinterpret_cast<double *>(z));
  if (!linear_smoothing<true>(pw, f * 2.0 / 3.0, fs, N, pw, reinterpret_cast<double *>(z), red)) {
    if (tid == 0) atomicOr_status(p.status, 2);
    return;
  }
  // ---- + |randn| * eps (:147-151), log, mirrored to an even sequence of N (:39-42) = input of the next FFT
  {
    double *zin = reinterpret_cast<double *>(z);
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const int k = tid + q * nth;
      if (k <= half) {
        const double v = pw[k] + fabs(randn_value(dpre[q])) * kEps;
        const double l = log(v);
        zin[rpad(k)] = l;
        if (k > 0 && k < half) zin[rpad(N - k)] = l;
      }
    }
    for (int k = tid + 5 * nth; k <= half; k += nth) {
      const double v = pw[k] + fabs(randn_value(draw[nwin + k])) * kEps;
      const double l = log(v);
      zin[rpad(k)] = l;
      if (k > 0 && k < half) zin[rpad(N - k)] = l;
    }
  }
  WB_SYNC();
  double2 *z2 = sfft_forward(z, o, lgc, p.tw);
  double2 *o2 = (z2 == A) ? B : A;
  // ---- liftering in the cepstrum domain (:28-37, 45-49); cos(2a) = 1 - 2 sin(a)^2 saves the cosine
  {
    double *zin = reinterpret_cast<double *>(o2);
    const double q1 = p.q1;
    // the lifters only scale floating-point values: quefrency through reciprocals, sin(pi a) by sinpi, 1/N exactly
    const double f_over_fs = f / fs, inv_n = 1.0 / N;
    rfft_unpack(z2, p.lg_fft, p.tw, [&](int k, double2 c) {
      double sl = 1.0, cl = (1.0 - 2.0 * q1) + 2.0 * q1;
      if (k > 0) {
        const double a = f_over_fs * k;          // f * quefrency
        const double sn = sinpi(a);
        sl = sn / (kPi * a);
        cl = (1.0 - 2.0 * q1) + 2.0 * q1 * (1.0 - 2.0 * sn * sn);
      }
      const double v = c.x * sl * cl * inv_n;
      zin[rpad(k)] = v;
      if (k > 0 && k < half) zin[rpad(N - k)] = v;
    });
  }
  WB_SYNC();
  double2 *z3 = sfft_forward(o2, z2, lgc, p.tw);
  if (!kCoded) {
    double *row = p.out + oidx * (size_t)p.out_stride;
    rfft_unpack(z3, p.lg_fft, p.tw, [&](int k, double2 c) { row[k] = exp(c.x); });
    return;
  }
  // ---- coded row: CodeSpectralEnvelope takes the log of the envelope (codec.cpp:288-289) -- the transform's real
  // part as it stands, the exp / log pair of the unfused path cancels -- interpolates it onto the mel grid (:121-122)
  // and runs DCTForCodec (:73-89) as one real FFT of fft_size / 2 points
  double2 *o3 = (z3 == A) ? B : A;
  double *lgs = reinterpret_cast<double *>(o3);   // half + 1 plain doubles
  rfft_unpack(z3, p.lg_fft, p.tw, [&](int k, double2 c) { lgs[k] = c.x; });
  WB_SYNC();
  {
    double *zin = reinterpret_cast<double *>(z3);
    const int bias = half / 2;
    for (int j = tid; j < bias; j += nth) {        // even samples ascending, odd samples descending (:77-81)
      const int a = 2 * j, b = half - 2 * j - 1;
      const int ka = __ldg(p.c_idx + a), kb = __ldg(p.c_idx + b);
      zin[rpad(j)] = lgs[ka] + __ldg(p.c_frac + a) * (lgs[ka + 1] - lgs[ka]);
      zin[rpad(j + bias)] = lgs[kb] + __ldg(p.c_frac + b) * (lgs[kb + 1] - lgs[kb]);
    }
  }
  WB_SYNC();
  const double2 *zc = sfft_forward(z3, o3, lgc - 1, p.tw);
  double *crow = p.c_out + oidx * (size_t)p.c_dims;
  const int dims = p.c_dims;
  const double cn = p.c_norm;
  rfft_unpack(zc, lgc, p.tw, [&](int d, double2 X) {     // :85-88
    if (d < dims) {
      const double2 w = __ldg(p.c_weight + d);
      crow[d] = (X.x * w.x - X.y * w.y) / cn;
    }
  });
}

#ifndef WB_EMU
__global__ void __launch_bounds__(128, 8) ct_frame_kernel(CtParams p) { ct_frame_body<false, false>(p); }
__global__ void __launch_bounds__(128, 8) ct_coded_kernel(CtParams p) { ct_frame_body<true, false>(p); }
__global__ void __launch_bounds__(128, 8) ct_frame_packed_kernel(CtParams p) { ct_frame_body<false, true>(p); }
__global__ void __launch_bounds__(128, 8) ct_coded_packed_kernel(CtParams p) { ct_frame_body<true, true>(p); }
#else
void ct_frame_kernel(CtParams p) { ct_frame_body<false, false>(p); }
void ct_coded_kernel(CtParams p) { ct_frame_body<true, false>(p); }
void ct_frame_packed_kernel(CtParams p) { ct_frame_body<false, true>(p); }
void ct_coded_packed_kernel(CtParams p) { ct_frame_body<true, true>(p); }
#endif

namespace {
// The utterances of a batch that share one CheapTrick option: their indices in the batch, ascending, and their frame
// counts.  ct_launch runs one launch sequence over them, reaching each row through the batch's own pointers.
struct UttGroup {
  std::vector<int> uid, f_len;
  int max_f_len = 0;
};
}  // namespace

// One launch sequence of one option (fft_size checked by stage_plan); row_stride: doubles per spectrogram row
// (0: fft_size / 2 + 1)
static int ct_launch(Ctx *ctx, const Batch &b, double q1, int fft_size, double *spectrogram, const CodecTables *coded,
                     double *coded_out, const UttGroup *group, int row_stride) {
  const int n_all = group ? (int)group->uid.size() : b.n;
  const int max_f_len = group ? group->max_f_len : b.max_f_len;
  if (n_all <= 0 || max_f_len <= 0) return 0;
  int lg = 0;
  while ((1 << lg) < fft_size) ++lg;
  const double f0_floor = 3.0 * b.fs / (fft_size - 3.0);  // GetF0FloorForCheapTrick, :196-198
  const int bins = fft_size / 2 + 1;
  // a frame draws at most (fft_size - 2) + bins numbers (2h+1 <= fft_size - 2 above the floor)
  const size_t max_per_frame = (size_t)fft_size + bins;
  const unsigned *table = rng_table_reserve(ctx, max_per_frame * (size_t)max_f_len);
  if (!table) return 2;
  // utterances per chunk so that the draw counts and offsets fit the budget (packed inputs: one pass, the packed stage
  // call cut its chunks by frames)
  const size_t per_utt_bytes = (size_t)b.f_stride * 8 + 64;
  int chunk = b.x_off ? n_all
                      : balanced_chunk(imin(n_all, 65535), (int)dmin(65535.0, (double)ctx->scratch_budget / (double)per_utt_bytes));
  // packed inputs: the launch's frames back to back in launch order, cum[k] before utterance k (the group's order)
  std::vector<long long> cum;
  if (b.x_off) {
    cum.assign(1, 0);
    for (int k = 0; k < n_all; ++k) {
      const int u = group ? group->uid[k] : k;
      cum.push_back(cum.back() + (b.f_off_host[u + 1] - b.f_off_host[u]));
    }
  }
  const size_t smem = ct_smem_bytes(fft_size);
#ifndef WB_EMU
  cudaFuncSetAttribute(ct_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(ct_coded_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (b.x_off) {
    cudaFuncSetAttribute(ct_frame_packed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(ct_coded_packed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
#endif
  const size_t n_tab = coded ? coded->idx.size() : 0, n_w = coded ? coded->weight.size() : 0;
  for (int u0 = 0; u0 < n_all; u0 += chunk) {
    const int n = imin(chunk, n_all - u0);
    ArenaPlan plan;
    const size_t slots = b.x_off ? (size_t)cum.back() : (size_t)n * b.f_stride;
    static_assert(WB_CT_FRAME_BYTES == 2 * sizeof(unsigned), "the per-frame arrays below");
    const size_t o_counts = plan.add(slots * sizeof(unsigned));
    const size_t o_offs = plan.add(slots * sizeof(unsigned));
    const size_t o_totals = plan.add((size_t)n * 4);
    const size_t o_cidx = plan.add(n_tab * 4 + 4), o_cfrac = plan.add(n_tab * 8 + 8), o_cw = plan.add(n_w * 16 + 16);
    const size_t o_group = plan.add(group ? (size_t)n * 8 : 0);
    const size_t o_cum = plan.add(b.x_off ? cum.size() * 8 : 0);
    unsigned char *blk = arena_block(ctx, plan.total);
    if (!blk) return 2;
    unsigned *counts = (unsigned *)(blk + o_counts), *offs = (unsigned *)(blk + o_offs);
    unsigned *totals = (unsigned *)(blk + o_totals);
    // a group keeps the batch's base pointers and reaches its utterances through uid; its frame counts are uploaded
    // in the launch's order, which is the order counts and offsets are laid out in
    const size_t base = group ? 0 : (size_t)u0;
    const int *uid = nullptr, *f_len = b.f_len + u0;
    if (group) {
      int *gd = (int *)(blk + o_group);
      int rc = dev_memcpy_h2d(ctx, gd, group->uid.data() + u0, (size_t)n * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, gd + n, group->f_len.data() + u0, (size_t)n * 4);
      if (rc) return rc;
      uid = gd; f_len = gd + n;
    }
    const long long *cum_dev = nullptr;
    if (b.x_off) {
      cum_dev = (const long long *)(blk + o_cum);
      const int rc = dev_memcpy_h2d(ctx, blk + o_cum, cum.data(), cum.size() * 8);
      if (rc) return rc;
    }
    const double *f0 = b.f0 + base * b.f_stride;
    const long long total_slots = (long long)slots;
    if (b.x_off) {
      if (total_slots)
        WB_LAUNCH_FLAT(ct_count_packed_kernel, dim3((unsigned)((total_slots + 255) / 256)), 256, 0, ctx->stream,
                       f0, b.f_off, cum_dev, n, b.fs, fft_size, f0_floor, uid, counts);
      scan_counts(ctx, counts, f_len, 0, nullptr, offs, totals, n, cum_dev);
    } else {
      WB_LAUNCH_FLAT(ct_count_kernel, dim3((unsigned)((total_slots + 255) / 256)), 256, 0, ctx->stream,
                     f0, f_len, b.f_stride, n, b.fs, fft_size, f0_floor, uid, counts);
      scan_counts(ctx, counts, f_len, b.f_stride, nullptr, offs, totals, n);
    }
    CtParams p;
    p.x = b.x + base * b.x_stride; p.x_len = b.x_len + base; p.x_stride = b.x_stride;
    p.time_axis = b.time_axis + base * b.f_stride; p.f0 = f0; p.f_len = f_len; p.uid = uid;
    p.x_off = b.x_off; p.cum = cum_dev; p.n_launch = n;
    // padded: one CTA per (frame, utterance) of the rows; packed: one per frame of the launch
    const dim3 grid = b.x_off ? dim3((unsigned)total_slots) : dim3((unsigned)max_f_len, (unsigned)n);
    p.f_stride = b.f_stride; p.fs = b.fs; p.fft_size = fft_size; p.lg_fft = lg;
    p.q1 = q1; p.f0_floor = f0_floor;
    p.draws = table; p.draw_off = offs;
    p.out_stride = row_stride > 0 ? row_stride : bins;
    // packed rows: the output pointers stay at frame 0 and f_off places each utterance
    const size_t out_base = b.f_off ? 0 : base * b.f_stride;
    p.f_off = b.f_off ? b.f_off + base : nullptr;
    p.out = spectrogram ? spectrogram + out_base * p.out_stride : nullptr;
    p.tw = ctx->twiddle; p.status = ctx->status_dev;
    p.c_dims = 0; p.c_idx = nullptr; p.c_frac = nullptr; p.c_weight = nullptr; p.c_norm = 1.0; p.c_out = nullptr;
    int ct_threads = 128;
    if (const char *e = getenv("WB_CT_THREADS")) ct_threads = atoi(e);
    if (coded) {
      int rc = dev_memcpy_h2d(ctx, blk + o_cidx, coded->idx.data(), n_tab * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_cfrac, coded->frac.data(), n_tab * 8);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_cw, coded->weight.data(), n_w * 16);
      if (rc) return rc;
      p.c_dims = coded->dims; p.c_idx = (const int *)(blk + o_cidx); p.c_frac = (const double *)(blk + o_cfrac);
      p.c_weight = (const double2 *)(blk + o_cw); p.c_norm = coded->norm;
      p.c_out = coded_out + out_base * coded->dims;
      if (b.x_off)
        WB_LAUNCH_COOP(ct_coded_packed_kernel, grid, ct_threads, smem, ctx->stream, p);
      else
        WB_LAUNCH_COOP(ct_coded_kernel, dim3((unsigned)max_f_len, (unsigned)n), ct_threads, smem, ctx->stream, p);
    } else if (b.x_off) {
      WB_LAUNCH_COOP(ct_frame_packed_kernel, grid, ct_threads, smem, ctx->stream, p);
    } else
    WB_LAUNCH_COOP(ct_frame_kernel, dim3((unsigned)max_f_len, (unsigned)n), ct_threads, smem, ctx->stream, p);
    int rc = dev_check(ctx, "cheaptrick");
    if (rc) return rc;
  }
  return 0;
}

int cheaptrick_run(Ctx *ctx, const StagePlan &stage, const Batch &b, int u0, double *out) {
  // one group per distinct (fft_size, q1), in order of first appearance
  std::vector<UttGroup> groups;
  for (int k = 0; k < b.n; ++k) {
    const int u = u0 + k;
    size_t g = 0;
    while (g < groups.size() && !(stage.fft_size[u0 + groups[g].uid[0]] == stage.fft_size[u] &&
                                  stage.q[u0 + groups[g].uid[0]] == stage.q[u]))
      ++g;
    if (g == groups.size()) groups.emplace_back();
    groups[g].uid.push_back(k);
    groups[g].f_len.push_back(stage.f_len[u]);
    groups[g].max_f_len = imax(groups[g].max_f_len, stage.f_len[u]);
  }
  int rc = 0;
  for (size_t g = 0; g < groups.size() && !rc; ++g) {
    const int u = u0 + groups[g].uid[0];
    // a batch of one option runs exactly as the one-option call
    const UttGroup *grp = groups.size() > 1 ? &groups[g] : nullptr;
    const double q1 = stage.q[u];
    const int fft_size = stage.fft_size[u];
    rc = stage.coded ? ct_launch(ctx, b, q1, fft_size, nullptr, &stage.tables[stage.table[u]], out, grp, 0)
                     : ct_launch(ctx, b, q1, fft_size, out, nullptr, nullptr, grp, stage.row);
  }
  return rc;
}

}  // namespace wb
