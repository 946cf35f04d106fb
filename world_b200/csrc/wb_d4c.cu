// wb_d4c.cu -- K-LT + K-D4C: band aperiodicity, one CTA per (utterance, frame), two passes.
//
// Replaces D4C() (d4c.cpp:342-403): pass A = D4CLoveTrain (:260-285, :227-252), pass B =
// D4CGeneralBody (:293-321) with GetStaticCentroid/GetCentroid (:90-140),
// GetSmoothedPowerSpectrum (:149-166), GetStaticGroupDelay (:172-188), GetCoarseAperiodicity
// (:194-225) and GetAperiodicity (:330-338).  Algorithm card: SURVEY.md A2.
//
// The reference's single randn stream runs through all of pass A and then all of pass B, so the
// driver counts pass-A draws, runs K-LT, counts pass-B draws of the frames K-LT selected
// (continuing after the pass-A total) and only then runs K-D4C.  std::sort + cumulative sum is
// restated as an order-statistic selection (k-th largest by bisection on the IEEE bit pattern)
// followed by a masked sum: the quantity needed is sum(smallest m)/sum(all).
// Every output row is written exactly once: by K-LT (default 1-1e-12 rows for unvoiced or
// rejected frames, d4c.cpp:323-328) or by K-D4C.
#include "wb_internal.h"
#include "wb_spectral.cuh"
#include <stdlib.h>

namespace wb {

struct D4cParams {
  const double *x; const int *x_len; int x_stride;
  const double *time_axis; const double *f0; const int *f_len; int f_stride;
  int fs;
  int ct_fft_size;          // rows have ct_fft_size/2+1 bins
  int lt_fft, lt_lg, b0, b1, b2;
  int d_fft, d_lg, n_ap, win_len, bd;
  double threshold;
  const double *nuttall;    // [win_len]
  const unsigned *draws; size_t draw_stride;
  const unsigned *off_a; unsigned *count_b; const unsigned *off_b;
  unsigned char *selected;  // [n][f_stride]
  int *slow_list; int *slow_count;   // frames whose window does not fit the fast body kernel (long windows, f0 near the floor)
  int pw_doubles;                    // doubles of the fast body kernel's power row (d4c_body_pw_doubles)
  double *out;
  const double2 *tw;
  const double2 *tw_body;   // compact twiddles of size d_fft (tw_sized_offset): the fast body kernel's
  int *status;
  // coded output (CodeAperiodicity, codec.cpp:228-238): with c_out set the kernels write the dB value at the c_n
  // band centres instead of the ct_fft_size/2+1 bins
  int c_n; const int *c_idx; const double *c_frac; double *c_out;
};

WB_KERNEL_PLAIN d4c_count_a_kernel(const double *__restrict__ f0, const int *__restrict__ f_len,
                                   int f_stride, int n_utts, int fs, unsigned *__restrict__ counts) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_utts * f_stride) return;
  const int u = (int)(g / f_stride), i = (int)(g % f_stride);
  unsigned c = 0;
  if (i < f_len[u] && f0[g] != 0.0) {
    const double f = dmax(f0[g], 40.0);
    c = (unsigned)(2 * round_half_away(3.0 * fs / f / 2.0) + 1);
  }
  counts[g] = c;
}

// F0-adaptive window + noise + weighted mean removal (d4c.cpp:21-83).  The windowed sample j goes to *pv(j), the
// window value to *pw(j) (callers choose the layout: packed FFT input, complex slot halves, ...).
// window_type 1 = Hanning, 2 = Blackman.  Ends with a barrier; every thread returns the same nwin.
template <class PV, class PW>
WB_DEV int d4c_windowed(const double *__restrict__ x, int x_len, int fs, double f, double pos,
                        int window_type, double ratio, const unsigned *__restrict__ draw,
                        PV pv, PW pw, double *red) {
  const int tid = WB_TID, nth = WB_NTH;
  const int h = round_half_away(ratio * fs / f / 2.0);
  const int nwin = 2 * h + 1;
  const int origin = round_half_away(pos * fs + 0.001);
  double s1 = 0.0, s2 = 0.0;
  for (int j = tid; j < nwin; j += nth) {
    const double position = (2.0 * (j - h) / ratio) / fs;
    double w;
    const double c1 = cos_small(kPi * position * f);
    if (window_type == 1)
      w = 0.5 * c1 + 0.5;
    else
      w = 0.42 + 0.5 * c1 + 0.08 * (2.0 * c1 * c1 - 1.0);   // cos(2a) = 2 cos(a)^2 - 1
    const int idx = imin(x_len - 1, imax(0, origin + j - h));
    const double v = x[idx] * w + randn_value(draw[j]) * 0.000001;  // kSafeGuardD4C
    *pv(j) = v;
    *pw(j) = w;
    s1 += v;
    s2 += w;
  }
  block_sum2(s1, s2, red);
  const double coef = s1 / s2;
  for (int j = tid; j < nwin; j += nth) *pv(j) = *pv(j) - *pw(j) * coef;
  WB_SYNC();
  return nwin;
}

// a frame D4C does not analyse (unvoiced, or LoveTrain says noise): 1 - 1e-12 in every bin (d4c.cpp:372-383);
// coded: 20 log10 of that at every band centre (interp1Q between equal nodes)
WB_DEV void d4c_fill_frame(const D4cParams &p, size_t fidx) {
  if (p.c_out) {
    const double v = 20 * log10(1.0 - kTiny);
    for (int b = WB_TID; b < p.c_n; b += WB_NTH) p.c_out[fidx * (size_t)p.c_n + b] = v;
    return;
  }
  const int bins = p.ct_fft_size / 2 + 1;
  double *row = p.out + fidx * (size_t)bins;
  for (int k = WB_TID; k < bins; k += WB_NTH) row[k] = 1.0 - kTiny;
}

// interp1 of the coarse aperiodicity (dB at 0, 3k, ..., fs/2) at bin k of the CheapTrick grid (d4c.cpp:330-338)
WB_DEV double d4c_bin_db(const double *coarse, int n_ap, int fs, int ct_fft_size, int k) {
  const int nx = n_ap + 2;
  const double xi = static_cast<double>(k) * fs / ct_fft_size;
  int idx = 0;  // number of axis points <= xi
  for (int j = 0; j < nx; ++j) {
    const double xj = (j == nx - 1) ? fs / 2.0 : j * 3000.0;
    idx += (xj <= xi) ? 1 : 0;
  }
  idx = imin(nx - 1, imax(1, idx));
  const double x0 = (idx - 1) * 3000.0;
  const double x1 = (idx == nx - 1) ? fs / 2.0 : idx * 3000.0;
  const double s = (xi - x0) / (x1 - x0);
  return coarse[idx - 1] + s * (coarse[idx] - coarse[idx - 1]);
}

// dB -> amplitude row (d4c.cpp:372-383), or the coded row: the dB values themselves, interp1Q'd onto the band centres
// (the 10^(y/20) / 20 log10 pair of the unfused path cancels)
template <bool kFastExp>
WB_DEV void d4c_write_frame(const D4cParams &p, size_t fidx, const double *coarse) {
  const int tid = WB_TID, nth = WB_NTH;
  const int bins = p.ct_fft_size / 2 + 1;
  if (p.c_out) {
    for (int b = tid; b < p.c_n; b += nth) {
      const int k = __ldg(p.c_idx + b);
      const double y0 = d4c_bin_db(coarse, p.n_ap, p.fs, p.ct_fft_size, k);
      const double dy = (k + 1 < bins) ? d4c_bin_db(coarse, p.n_ap, p.fs, p.ct_fft_size, k + 1) - y0 : 0.0;
      p.c_out[fidx * (size_t)p.c_n + b] = y0 + dy * __ldg(p.c_frac + b);
    }
    return;
  }
  double *row = p.out + fidx * (size_t)bins;
  for (int k = tid; k < bins; k += nth) {
    const double y = d4c_bin_db(coarse, p.n_ap, p.fs, p.ct_fft_size, k);
    row[k] = kFastExp ? exp(y * 0.11512925464970228420)   // 10^(y/20) = e^(y ln10 / 20)
                      : pow(10.0, y / 20.0);
  }
}

// ------------------------------------------------------------------ pass A: LoveTrain
WB_KERNEL(128, 4) d4c_lovetrain_kernel(D4cParams p) {
  WB_DYN_SMEM(double2, smem2);
  const int tid = WB_TID, nth = WB_NTH;
  const int u = blockIdx.y, i = blockIdx.x;
  if (i >= p.f_len[u]) return;
  const size_t fidx = (size_t)u * p.f_stride + i;
  const double f0 = p.f0[fidx];
  if (f0 == 0.0) {
    d4c_fill_frame(p, fidx);
    if (tid == 0) { p.selected[fidx] = 0; p.count_b[fidx] = 0; }
    return;
  }
  const int N = p.lt_fft, half = N / 2;
  const int slots = WB_FPAD_SLOTS(half);
  double2 *A = smem2, *B = smem2 + slots;         // padded ping-pong pair of N/2 complex slots (wb_fft.cuh)
  double *red = reinterpret_cast<double *>(B + slots);
  double *za = reinterpret_cast<double *>(A), *win = reinterpret_cast<double *>(B);
  const double f = dmax(f0, 40.0);
  const double *x = p.x + (size_t)u * p.x_stride;
  const unsigned *draw = p.draws + (size_t)u * p.draw_stride + p.off_a[fidx];
  const int nwin = d4c_windowed(x, p.x_len[u], p.fs, f, p.time_axis[fidx], 2, 3.0, draw,
                                [&](int j) { return za + rpad(j); }, [&](int j) { return win + j; }, red);
  for (int j = nwin + tid; j < N; j += nth) za[rpad(j)] = 0.0;
  WB_SYNC();
  const double2 *z = sfft_forward(A, B, p.lt_lg - 1, p.tw);
  // cumulative power b0+1..b1 and b0+1..b2 (d4c.cpp:241-249), summed while the real FFT is unpacked
  double s_lo = 0.0, s_hi = 0.0;
  const int lo = p.b0 + 1, hi_end = imin(p.b2, half), b1 = p.b1;
  rfft_unpack(z, p.lt_lg, p.tw, [&](int k, double2 c) {
    if (k >= lo && k <= hi_end) {
      const double pw = c.x * c.x + c.y * c.y;
      s_hi += pw;
      if (k <= b1) s_lo += pw;
    }
  });
  block_sum2(s_lo, s_hi, red);
  const double ap0 = s_lo / s_hi;
  const bool sel = ap0 > p.threshold;  // d4c.cpp:386
  if (!sel) d4c_fill_frame(p, fidx);
  if (tid == 0) {
    p.selected[fidx] = sel ? 1 : 0;
    unsigned c = 0;
    if (sel) {
      const double fb = dmax(47.0, f0);  // kFloorF0D4C
      c = 3u * (unsigned)(2 * round_half_away(4.0 * p.fs / fb / 2.0) + 1);
    }
    p.count_b[fidx] = c;
  }
}

// k-th largest (1-based) of the non-negative doubles a[0..n): bisection on the IEEE bit pattern,
// two bits per round (three pivots counted at once), one barrier per round (the per-warp count
// slots alternate between two halves of `red`, so a round never overwrites what a slow warp of
// the previous round still reads).  red: >= 2 * 2 * 33 ints.
WB_DEV double select_kth_largest(const double *a, int n, int kth, double *red) {
  const int tid = WB_TID, nth = WB_NTH;
  unsigned long long pat = 0ull;
  int round = 0;
  // `red` is the scratch the block reductions read without a trailing barrier: a warp still summing the
  // previous block_sum's partials must not see round 0's counts (found by compute-sanitizer racecheck)
  WB_SYNC();
  for (int bit = 62; bit >= 0; bit -= 2, ++round) {
    const bool two = bit >= 1;
    const unsigned long long hi_bit = 1ull << bit, lo_bit = two ? (1ull << (bit - 1)) : 0ull;
    const unsigned long long p01 = pat | lo_bit, p10 = pat | hi_bit, p11 = pat | hi_bit | lo_bit;
    int c01 = 0, c10 = 0, c11 = 0;
        for (int j = tid; j < n; j += nth) {
      const double v = a[j];
      unsigned long long bits;
#ifdef WB_EMU
      memcpy(&bits, &v, 8);
#else
      bits = (unsigned long long)__double_as_longlong(v);
#endif
      c01 += (bits >= p01) ? 1 : 0;
      c10 += (bits >= p10) ? 1 : 0;
      c11 += (bits >= p11) ? 1 : 0;
    }
#ifndef WB_EMU
    int *ired = reinterpret_cast<int *>(red) + (round & 1) * 2 * 33;
    const int packed = __reduce_add_sync(0xffffffffu, c01 | (c10 << 16));
    c11 = __reduce_add_sync(0xffffffffu, c11);
    const int lane = tid & 31, w = tid >> 5, nw = (nth + 31) >> 5;
    if (lane == 0) { ired[w] = packed; ired[33 + w] = c11; }
    __syncthreads();
    int sp = 0, s11 = 0;
    for (int i = 0; i < nw; ++i) { sp += ired[i]; s11 += ired[33 + i]; }
    c01 = sp & 0xffff; c10 = sp >> 16; c11 = s11;
#endif
    // largest pattern whose ">= count" still reaches kth
    if (two && c11 >= kth) pat = p11;
    else if (c10 >= kth) pat = p10;
    else if (two && c01 >= kth) pat = p01;
  }
#ifndef WB_EMU
  __syncthreads();
#endif
  double r;
#ifdef WB_EMU
  memcpy(&r, &pat, 8);
#else
  r = __longlong_as_double((long long)pat);
#endif
  return r;
}

// The same order statistic through a short candidate list (GPU only; round 1's bisection -- 32 rounds over all n
// values with a barrier each -- was a large share of the body kernel's instructions):
//   1. every thread takes the maximum of the values it owns (a[tid], a[tid + nth], ...);
//   2. L = the kth largest of those maxima (of 32 maxima over four threads each when kth <= 32) is a lower bound of
//      the answer (the kth largest maxima are kth distinct elements >= L), and for spectra -- no long runs of equal
//      values -- only a few more than kth elements reach it;
//   3. the elements >= L are collected (shared-memory counter) and ranked against each other exactly.
// Comparisons run on the IEEE bit patterns (a total order on the non-negative values, ties broken by index), so the
// value returned is the one the bisection returns.  Returns false to every thread -- nothing useful in *out -- when
// kth > nth or more than WB_SEL_CAP elements reach L; the caller then falls back to the bisection.
// scratch: nth + WB_SEL_CAP + 4 64-bit words of shared memory.  Contains barriers.
#define WB_SEL_CAP 256
WB_DEV bool select_kth_largest_fast(const double *a, int n, int kth, unsigned long long *scratch, double *out) {
#ifdef WB_EMU
  (void)a; (void)n; (void)kth; (void)scratch; (void)out;
  return false;   // one emulated thread: the bisection is the reference semantics anyway
#else
  const int tid = threadIdx.x, nth = blockDim.x;
  if (kth < 1 || kth > nth || kth > n) return false;
  unsigned long long *cand = scratch + nth + 4;
  unsigned *counter = reinterpret_cast<unsigned *>(scratch + nth + 1);
  unsigned long long mx = 0ull;
  for (int j = tid; j < n; j += nth) {
    const unsigned long long k = (unsigned long long)__double_as_longlong(a[j]);
    mx = k > mx ? k : mx;
  }
  scratch[tid] = mx;
  if (tid == 0) *counter = 0u;
  __syncthreads();
  if (kth <= 32) {
    // 32 maxima (lane l of warp 0: the threads l, l + 32, ...) are enough for a lower bound when kth <= 32: the bound
    // is a little lower, a few more elements pass it, and the ranking is 32 shuffles in one warp instead of nth
    // shared-memory reads in every thread
    if (tid < 32) {
      unsigned long long m32 = 0ull;
      for (int t = tid; t < nth; t += 32) { const unsigned long long kt = scratch[t]; m32 = kt > m32 ? kt : m32; }
      int r = 0;
      for (int t = 0; t < 32; ++t) {
        const unsigned long long kt = __shfl_sync(0xffffffffu, m32, t);
        r += (kt > m32 || (kt == m32 && t < tid)) ? 1 : 0;
      }
      if (r == kth - 1) scratch[nth] = m32;
    }
  } else {
    int r = 0;
    for (int t = 0; t < nth; ++t) {
      const unsigned long long kt = scratch[t];
      r += (kt > mx || (kt == mx && t < tid)) ? 1 : 0;
    }
    if (r == kth - 1) scratch[nth] = mx;
  }
  __syncthreads();
  const unsigned long long L = scratch[nth];
  for (int j = tid; j < n; j += nth) {
    const unsigned long long k = (unsigned long long)__double_as_longlong(a[j]);
    if (k >= L) {
      const unsigned at = atomicAdd(counter, 1u);
      if (at < WB_SEL_CAP) cand[at] = k;
    }
  }
  __syncthreads();
  const int c = (int)*counter;
  if (c > WB_SEL_CAP) return false;
  for (int i = tid; i < c; i += nth) {
    const unsigned long long ki = cand[i];
    int r = 0;
    for (int t = 0; t < c; ++t) {
      const unsigned long long kt = cand[t];
      r += (kt > ki || (kt == ki && t < i)) ? 1 : 0;
    }
    if (r == kth - 1) scratch[nth + 2] = ki;
  }
  __syncthreads();
  *out = __longlong_as_double((long long)scratch[nth + 2]);
  return true;
#endif
}

// ------------------------------------------------------------------ pass B: general body
// One CTA of d_fft / 16 threads per selected frame.  Shared memory: ONE padded buffer of d_fft / 2 complex slots
// (in-place self-sorting FFT, wb_fft.cuh: one radix-8 butterfly per thread and pass), the centroid row, the power
// row, reduction scratch -- 36.5 KB at 16 kHz, six CTAs per SM.  Every transform is a complex FFT of d_fft / 2:
//   * power spectrum and the n_ap band spectra: real FFTs, two samples per slot, unpacked on the fly;
//   * centroid: the reference's two real FFTs of v and (n+1) v = one complex FFT of d_fft of z = v + j (n+1) v, done
//     here as its two decimation-in-frequency halves -- even bins from z[n] + z[n + d_fft/2], odd bins from
//     (z[n] - z[n + d_fft/2]) W^n -- one after the other in the same buffer (bins k and d_fft - k, which the
//     split of the two real spectra pairs up, have the same parity).  The windowed signal waits in the power row.
// Frames whose window is longer than the power row (d4c_body_pw_doubles: f0 near the 47 Hz floor) go to slow_list
// and are done by d4c_body_slow_kernel (the round-1 body on the in-place DIT FFT, any window length), as is every
// frame when d_fft is above 4096 or below 512 (this kernel's thread count would not fit a CTA, or fill a warp).
// Doubles of the power row.  It also holds the windowed signal of the centroid transforms, whose longest window (f0
// at the 47 Hz floor, ratio 4) is up to twice d_fft / 2 + 1; shared memory per CTA decides how many CTAs an SM holds
// and the kernel is latency bound (sizing the row for the longest window costs a CTA per SM at 48 kHz), so the row grows only as far as the CTA count of the minimal layout allows.  Frames with
// a longer window (f0 below ~54 Hz at 16 kHz, ~75 Hz at 48 kHz) go to slow_list / d4c_body_slow_kernel.
WB_HD inline size_t d4c_body_smem_bytes_for(int d_fft, int pw_doubles, int n_ap, int threads) {
  return (size_t)WB_FPAD_SLOTS(d_fft / 2) * sizeof(double2) +
         (size_t)((d_fft / 2 + 1) + pw_doubles + WB_RED_DOUBLES + (threads + 1) + (n_ap + 2) + 2) * sizeof(double);
}
WB_HD inline int d4c_body_pw_doubles(int d_fft, int fs, int n_ap, int threads) {
  const int nwin_max = 2 * round_half_away(4.0 * fs / 47.0 / 2.0) + 1;
  const int half1 = d_fft / 2 + 1;
  const size_t per_sm = (size_t)227 * 1024, reserved = 1024;
  const size_t smem_min = d4c_body_smem_bytes_for(d_fft, half1, n_ap, threads);
  const size_t ctas = per_sm / (smem_min + reserved);
  if (ctas == 0) return half1;
  const size_t slack = (per_sm / ctas - reserved - smem_min) / sizeof(double);
  const int grown = half1 + (int)slack - 2;
  return imax(half1, imin(nwin_max + 1, grown));
}

// kLg = log2(d_fft), 9..12: the transforms are sfft_forward_fixed at compile-time size on d_fft / 16 threads, with the
// compact twiddle table p.tw_body of size d_fft (every twiddle the frame reads: the passes, the real-FFT unpack and the
// centroid's DIF split)
template <int kLg>
WB_DEV void d4c_body_frame(const D4cParams &p) {
  WB_DYN_SMEM(double2, smem2);
  const int tid = WB_TID, nth = WB_NTH;
  const int u = blockIdx.y, i = blockIdx.x;
  if (i >= p.f_len[u]) return;
  const size_t fidx = (size_t)u * p.f_stride + i;
  if (!p.selected[fidx]) return;
  constexpr int N = 1 << kLg, half = N / 2;
  const int fs = p.fs;
  const double2 *__restrict__ twc = p.tw_body;
  const int slots = WB_FPAD_SLOTS(half);
  double2 *P = smem2;
  double *pd = reinterpret_cast<double *>(P);            // the same buffer as 2 * slots plain doubles
  double *cent = reinterpret_cast<double *>(P + slots);  // half + 1
  const int pw_doubles = p.pw_doubles;
  double *pw = cent + (half + 1);          // power row (half + 1); the windowed signal during the centroid transforms
  double *red = pw + pw_doubles;           // WB_RED_DOUBLES
  double *red_big = red + WB_RED_DOUBLES;  // nth + 1
  double *coarse = red_big + (nth + 1);    // n_ap + 2
  double *wv = pd;                         // window values while a window is built: the FFT buffer is idle then

  const double f = dmax(47.0, p.f0[fidx]);
  const double t = p.time_axis[fidx];
  {
    const int nwin4 = 2 * round_half_away(4.0 * fs / f / 2.0) + 1;   // both ratio-4 windows (d4c_windowed)
    if (nwin4 > pw_doubles || nwin4 > 2 * slots) {   // long window: the any-length kernel takes the frame
      if (tid == 0) {
#ifdef WB_EMU
        const int at = (*p.slow_count)++;
#else
        const int at = atomicAdd(p.slow_count, 1);
#endif
        p.slow_list[at] = (int)(u * p.f_stride + i);
      }
      return;
    }
  }
  const double *x = p.x + (size_t)u * p.x_stride;
  const int x_len = p.x_len[u];
  const unsigned *draw = p.draws + (size_t)u * p.draw_stride + p.off_b[fidx];

  // ---- static centroid = centroid(t - 1/4f) + centroid(t + 1/4f)   (d4c.cpp:90-140)
  for (int pass = 0; pass < 2; ++pass) {
    const double pos = pass == 0 ? t - 0.25 / f : t + 0.25 / f;
    const int nwin = d4c_windowed(x, x_len, fs, f, pos, 2, 4.0, draw, [&](int j) { return pw + j; },
                                  [&](int j) { return wv + j; }, red);
    draw += nwin;
    double sq = 0.0;
    for (int j = tid; j < nwin; j += nth) { const double v = pw[j]; sq += v * v; }
    const double rt = sqrt(block_sum(sq, red));
    for (int part = 0; part < 2; ++part) {
      // input of the half transform: z[n] = v[n] / rt * (1 + j (n + 1)), n < nwin
      for (int n = tid; n < half; n += nth) {
        double2 z0 = make_double2(0.0, 0.0), z1 = make_double2(0.0, 0.0);
        if (n < nwin) { const double v = pw[n] / rt; z0 = make_double2(v, v * (n + 1.0)); }
        if (n + half < nwin) { const double v = pw[n + half] / rt; z1 = make_double2(v, v * (n + half + 1.0)); }
        P[fpad(n)] = part == 0 ? cadd(z0, z1) : cmul(__ldg(&twc[n]), csub(z0, z1));
      }
      WB_SYNC();
      sfft_forward_fixed<kLg - 1>(P, twc);
      // bins k = 2 m + part; partner N - k = 2 (half - m - part) + part.  A = spectrum of v, B = of (n+1) v
      for (int m = tid; 2 * m + part <= half; m += nth) {
        const double2 zp = P[fpad(m)], zq = P[fpad((half - m - part) & (half - 1))];
        const double ar = 0.5 * (zp.x + zq.x), ai = 0.5 * (zp.y - zq.y);
        const double br = 0.5 * (zp.y + zq.y), bi = -0.5 * (zp.x - zq.x);
        const double c = br * ar + ai * bi;
        const int k = 2 * m + part;
        cent[k] = pass == 0 ? c : cent[k] + c;
      }
      WB_SYNC();
    }
  }
  dc_correction(cent, f, fs, N, pd);

  // ---- smoothed power spectrum (d4c.cpp:149-166)
  {
    const int nwin = d4c_windowed(x, x_len, fs, f, t, 1, 4.0, draw, [&](int j) { return pd + rpad(j); },
                                  [&](int j) { return pw + j; }, red);
    for (int j = nwin + tid; j < N; j += nth) pd[rpad(j)] = 0.0;
    WB_SYNC();
    sfft_forward_fixed<kLg - 1>(P, twc);
    rfft_unpack(P, kLg, twc, [&](int k, double2 c) { pw[k] = c.x * c.x + c.y * c.y; }, kLg);
    WB_SYNC();
    dc_correction(pw, f, fs, N, pd);
    if (!linear_smoothing<false>(pw, f, fs, N, pw, pd, red_big)) {
      if (tid == 0) atomicOr_status(p.status, 2);
      return;
    }
  }
  // ---- static group delay (d4c.cpp:172-188): g = cent / pw, two smoothers
  for (int k = tid; k <= half; k += nth) pw[k] = cent[k] / pw[k];
  WB_SYNC();
  bool ok = linear_smoothing<false>(pw, f / 2.0, fs, N, pw, pd, red_big);
  ok = ok && linear_smoothing<false>(pw, f, fs, N, cent, pd, red_big);
  if (!ok) {
    if (tid == 0) atomicOr_status(p.status, 2);
    return;
  }
  for (int k = tid; k <= half; k += nth) pw[k] = pw[k] - cent[k];
  WB_SYNC();

  // ---- coarse aperiodicity per 3 kHz band (d4c.cpp:194-225)
  const int half_w = p.win_len / 2;
  for (int b = 0; b < p.n_ap; ++b) {
    const int center = static_cast<int>(3000.0 * (b + 1) * N / fs);
    for (int j = tid; j < N; j += nth)
      pd[rpad(j)] = (j <= half_w * 2) ? pw[center - half_w + j] * __ldg(&p.nuttall[j]) : 0.0;
    WB_SYNC();
    sfft_forward_fixed<kLg - 1>(P, twc);
    double tot = 0.0;
    rfft_unpack(P, kLg, twc, [&](int k, double2 c) {
      const double v = c.x * c.x + c.y * c.y;
      cent[k] = v;
      tot += v;
    }, kLg);
    tot = block_sum(tot, red);  // contains the barrier that publishes cent[]
    const int n_small = half - p.bd;  // entries in the sorted prefix, index half-bd-1 inclusive
    double kth;
    // the FFT buffer is idle: candidate scratch (nth + WB_SEL_CAP + 4 words <= 2 * slots)
    if (!select_kth_largest_fast(cent, half + 1, p.bd + 1, reinterpret_cast<unsigned long long *>(pd), &kth))
      kth = select_kth_largest(cent, half + 1, p.bd + 1, red);
    double below = 0.0, n_below = 0.0;   // the count is exact in a double: one reduction for both
    for (int k = tid; k <= half; k += nth)
      if (cent[k] < kth) { below += cent[k]; n_below += 1.0; }
    block_sum2(below, n_below, red);
    const double small = below + (double)(n_small - (int)n_below) * kth;
    if (tid == 0) {
      const double c = 10.0 * log10(small / tot);
      coarse[b + 1] = dmin(0.0, c + (f - 100.0) / 50.0);  // d4c.cpp:314-316
    }
    WB_SYNC();
  }
  if (tid == 0) { coarse[0] = -60.0; coarse[p.n_ap + 1] = -kTiny; }
  WB_SYNC();

  // ---- interp1 onto the CheapTrick frequency grid, dB -> amplitude (d4c.cpp:330-338, 372-383)
  d4c_write_frame<true>(p, fidx, coarse);
}

// d_fft / 16 threads; the register budget (80) of 768 threads per SM -- six CTAs at 16 kHz, as many as the shared
// memory holds
template <int kLg>
WB_KERNEL(1 << (kLg - 4), 768 >> (kLg - 4)) d4c_body_kernel_lg(D4cParams p) { d4c_body_frame<kLg>(p); }

typedef void (*D4cBodyKernel)(D4cParams);
// nullptr: no fast body kernel at this size (d_fft below 512 or above 4096)
static D4cBodyKernel d4c_body_kernel_for(int d_lg) {
  switch (d_lg) {
    case 9: return d4c_body_kernel_lg<9>;
    case 10: return d4c_body_kernel_lg<10>;
    case 11: return d4c_body_kernel_lg<11>;
    case 12: return d4c_body_kernel_lg<12>;
    default: return nullptr;
  }
}

// ------------------------------------------------------------------ pass B, any window length (round-1 body, in-place DIT FFT)
// Persistent kernel over slow_list (frames the fast kernel handed over); with d_fft > 4096 (fs above 48.1 kHz: the
// fast kernel's thread count would exceed a CTA) the driver puts every selected frame on the list instead.
WB_DEV void d4c_body_slow_frame(const D4cParams &p, int u, int i, double *smem) {
  const int tid = WB_TID, nth = WB_NTH;
  const size_t fidx = (size_t)u * p.f_stride + i;
  const int N = p.d_fft, half = N / 2, fs = p.fs;
  double *zb = smem;                       // 2N (+2): complex FFT buffer / smoothing scratch
  double *cent = zb + 2 * N + 2;           // half + 1
  double *pw = cent + (half + 1);          // half + 1
  double *red = pw + (half + 1);           // WB_RED_DOUBLES
  double *red_big = red + WB_RED_DOUBLES;  // nth + 1
  double *coarse = red_big + (nth + 1);    // n_ap + 2
  double2 *z = reinterpret_cast<double2 *>(zb);

  const double f = dmax(47.0, p.f0[fidx]);
  const double t = p.time_axis[fidx];
  const double *x = p.x + (size_t)u * p.x_stride;
  const int x_len = p.x_len[u];
  const unsigned *draw = p.draws + (size_t)u * p.draw_stride + p.off_b[fidx];

  // ---- static centroid = centroid(t - 1/4f) + centroid(t + 1/4f)   (d4c.cpp:90-140)
  for (int pass = 0; pass < 2; ++pass) {
    const double pos = pass == 0 ? t - 0.25 / f : t + 0.25 / f;
    // re = windowed sample, im = window (scratch) while the mean is removed
    const int nwin = d4c_windowed(x, x_len, fs, f, pos, 2, 4.0, draw, [&](int j) { return zb + 2 * j; },
                                  [&](int j) { return zb + 2 * j + 1; }, red);
    draw += nwin;
    double sq = 0.0;
        for (int j = tid; j < nwin; j += nth) sq += z[j].x * z[j].x;
    const double rt = sqrt(block_sum(sq, red));
        for (int j = tid; j < N; j += nth) {
      if (j < nwin) {
        const double v = z[j].x / rt;
        z[j] = make_double2(v, v * (j + 1.0));
      } else {
        z[j] = make_double2(0.0, 0.0);
      }
    }
    WB_SYNC();
    cfft_forward(z, p.d_lg, p.tw);
        for (int k = tid; k <= half; k += nth) {
      double2 A, B;
      split_pair(z, N, k, A, B);
      const double c = B.x * A.x + A.y * B.y;
      cent[k] = pass == 0 ? c : cent[k] + c;
    }
    WB_SYNC();
  }
  dc_correction(cent, f, fs, N, zb);

  // ---- smoothed power spectrum (d4c.cpp:149-166)
  {
    const int nwin = d4c_windowed(x, x_len, fs, f, t, 1, 4.0, draw, [&](int j) { return zb + j; },
                                  [&](int j) { return zb + N + 2 + j; }, red);
        for (int j = nwin + tid; j < N + 2; j += nth) zb[j] = 0.0;
    WB_SYNC();
    rfft_forward(zb, p.d_lg, p.tw);
        for (int k = tid; k <= half; k += nth) { const double2 c = z[k]; pw[k] = c.x * c.x + c.y * c.y; }
    WB_SYNC();
    dc_correction(pw, f, fs, N, zb);
    if (!linear_smoothing<false>(pw, f, fs, N, pw, zb, red_big)) {
      if (tid == 0) atomicOr_status(p.status, 2);
      return;
    }
  }
  // ---- static group delay (d4c.cpp:172-188): g = cent / pw, two smoothers
    for (int k = tid; k <= half; k += nth) pw[k] = cent[k] / pw[k];
  WB_SYNC();
  bool ok = linear_smoothing<false>(pw, f / 2.0, fs, N, pw, zb, red_big);
  ok = ok && linear_smoothing<false>(pw, f, fs, N, cent, zb, red_big);
  if (!ok) {
    if (tid == 0) atomicOr_status(p.status, 2);
    return;
  }
    for (int k = tid; k <= half; k += nth) pw[k] = pw[k] - cent[k];
  WB_SYNC();

  // ---- coarse aperiodicity per 3 kHz band (d4c.cpp:194-225)
  const int half_w = p.win_len / 2;
  for (int b = 0; b < p.n_ap; ++b) {
    const int center = static_cast<int>(3000.0 * (b + 1) * N / fs);
        for (int j = tid; j < N + 2; j += nth)
      zb[j] = (j <= half_w * 2) ? pw[center - half_w + j] * __ldg(&p.nuttall[j]) : 0.0;
    WB_SYNC();
    rfft_forward(zb, p.d_lg, p.tw);
    double tot = 0.0;
        for (int k = tid; k <= half; k += nth) {
      const double2 c = z[k];
      const double v = c.x * c.x + c.y * c.y;
      cent[k] = v;
      tot += v;
    }
    tot = block_sum(tot, red);  // contains the barrier that publishes cent[]
    const int n_small = half - p.bd;  // entries in the sorted prefix, index half-bd-1 inclusive
    const double kth = select_kth_largest(cent, half + 1, p.bd + 1, red);
    double below = 0.0;
    int n_below = 0;
        for (int k = tid; k <= half; k += nth)
      if (cent[k] < kth) { below += cent[k]; ++n_below; }
    below = block_sum(below, red);
    n_below = block_sum_int(n_below, red);
    const double small = below + (double)(n_small - n_below) * kth;
    if (tid == 0) {
      const double c = 10.0 * log10(small / tot);
      coarse[b + 1] = dmin(0.0, c + (f - 100.0) / 50.0);  // d4c.cpp:314-316
    }
    WB_SYNC();
  }
  if (tid == 0) { coarse[0] = -60.0; coarse[p.n_ap + 1] = -kTiny; }
  WB_SYNC();

  // ---- interp1 onto the CheapTrick frequency grid, dB -> amplitude (d4c.cpp:330-338, 372-383)
  d4c_write_frame<false>(p, fidx, coarse);
}

WB_KERNEL(256, 2) d4c_body_slow_kernel(D4cParams p) {
  WB_DYN_SMEM(double, smem);
  const int count = *p.slow_count;
  for (int at = blockIdx.x; at < count; at += gridDim.x) {
    const int g = p.slow_list[at];
    d4c_body_slow_frame(p, g / p.f_stride, g % p.f_stride, smem);
    WB_SYNC();   // the next frame reuses the shared buffers
  }
}

// no fast body kernel at this d_fft: every selected frame goes through the list
WB_KERNEL_PLAIN d4c_list_all_kernel(D4cParams p, int n_utts) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_utts * p.f_stride) return;
  const int u = (int)(g / p.f_stride), i = (int)(g % p.f_stride);
  if (i >= p.f_len[u] || !p.selected[g]) return;
#ifdef WB_EMU
  const int at = (*p.slow_count)++;
#else
  const int at = atomicAdd(p.slow_count, 1);
#endif
  p.slow_list[at] = (int)g;
}

int d4c_run(Ctx *ctx, const Batch &b, int fft_size, double threshold, double *aperiodicity,
            const CodecTables *coded, double *coded_out) {
  if (b.n <= 0 || b.max_f_len <= 0) return 0;
  if (coded && coded->dims == 0) return 0;   // below 12 kHz the coded row is empty (codec.cpp:216-219)
  const int fs = b.fs;
  D4cParams p;
  memset(&p, 0, sizeof(p));
  p.fs = fs;
  p.ct_fft_size = fft_size;
  p.threshold = threshold;
  // sizes with the reference's expressions (host libm), d4c.cpp:350-365 and :262-272
  p.d_fft = static_cast<int>(pow(2.0, 1.0 + static_cast<int>(log(4.0 * fs / 47.0 + 1) / kLog2)));
  p.lt_fft = static_cast<int>(pow(2.0, 1.0 + static_cast<int>(log(3.0 * fs / 40.0 + 1) / kLog2)));
  for (p.d_lg = 0; (1 << p.d_lg) < p.d_fft; ++p.d_lg) {}
  for (p.lt_lg = 0; (1 << p.lt_lg) < p.lt_fft; ++p.lt_lg) {}
  if (fft_size < 4) {
    ctx->last_error = "D4C: fft_size must be at least 4";
    return 3;
  }
  if (p.d_fft > WB_TW_N || p.lt_fft > WB_TW_N) {
    ctx->last_error = "D4C: sampling rate too high for the on-chip FFT (fft > 8192)";
    return 3;
  }
  p.n_ap = static_cast<int>(dmin(15000.0, fs / 2.0 - 3000.0) / 3000.0);
  if (p.n_ap < 0) p.n_ap = 0;
  p.win_len = static_cast<int>(3000.0 * p.d_fft / fs) * 2 + 1;
  p.bd = round_half_away(p.d_fft * 8.0 / p.win_len);
  p.b0 = static_cast<int>(ceil(100.0 * p.lt_fft / fs));
  p.b1 = static_cast<int>(ceil(4000.0 * p.lt_fft / fs));
  p.b2 = static_cast<int>(ceil(7900.0 * p.lt_fft / fs));
  const int bins = fft_size / 2 + 1;

  // Nuttall window of the band analysis (common.cpp:113-121), host libm like the reference
  double *nuttall_host = new double[p.win_len];
  for (int i = 0; i < p.win_len; ++i) {
    const double tmp = i / (p.win_len - 1.0);
    nuttall_host[i] = 0.355768 - 0.487396 * cos(2.0 * kPi * tmp) + 0.144232 * cos(4.0 * kPi * tmp) -
                      0.012604 * cos(6.0 * kPi * tmp);
  }

  const size_t max_a = (size_t)(2 * round_half_away(3.0 * fs / 40.0 / 2.0) + 1);
  const size_t max_b = 3 * (size_t)(2 * round_half_away(4.0 * fs / 47.0 / 2.0) + 1);
  const size_t draw_stride_full = (max_a + max_b) * (size_t)b.max_f_len;
  const size_t per_utt_bytes = draw_stride_full * 4 + (size_t)b.f_stride * 28 + 64;
  int chunk = balanced_chunk(imin(b.n, 65535), (int)dmin(65535.0, (double)ctx->scratch_budget / (double)per_utt_bytes));
  // fast body kernel: one radix-8 butterfly per thread in the passes of the d_fft / 2 complex transforms; at d_fft
  // above 4096 its thread count would exceed a CTA, below 512 a warp
  const D4cBodyKernel d4c_body_kernel = d4c_body_kernel_for(p.d_lg);
  const bool all_slow = d4c_body_kernel == nullptr;
  int body_threads = p.d_fft / 16, lt_threads = 128, slow_threads = 128;
  if (const char *e = getenv("WB_LT_THREADS")) lt_threads = atoi(e);
  const size_t smem_lt = (size_t)2 * WB_FPAD_SLOTS(p.lt_fft / 2) * sizeof(double2) + WB_RED_DOUBLES * sizeof(double);
  p.pw_doubles = d4c_body_pw_doubles(p.d_fft, fs, p.n_ap, body_threads);
  const size_t smem_body = d4c_body_smem_bytes_for(p.d_fft, p.pw_doubles, p.n_ap, body_threads);
  const size_t smem_slow = (size_t)((2 * p.d_fft + 2) + 2 * (p.d_fft / 2 + 1) + WB_RED_DOUBLES +
                                    (slow_threads + 1) + (p.n_ap + 2) + 2) * sizeof(double);
#ifndef WB_EMU
  cudaFuncSetAttribute(d4c_lovetrain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_lt);
  if (!all_slow) cudaFuncSetAttribute(d4c_body_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_body);
  cudaFuncSetAttribute(d4c_body_slow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_slow);
#endif
  int rc = 0;
  for (int u0 = 0; u0 < b.n && rc == 0; u0 += chunk) {
    const int n = imin(chunk, b.n - u0);
    const size_t slots = (size_t)n * b.f_stride;
    ArenaPlan plan;
    const size_t o_ca = plan.add(slots * 4), o_oa = plan.add(slots * 4);
    const size_t o_cb = plan.add(slots * 4), o_ob = plan.add(slots * 4);
    const size_t o_ta = plan.add((size_t)n * 4), o_tab = plan.add((size_t)n * 4);
    const size_t o_sel = plan.add(slots), o_nut = plan.add((size_t)p.win_len * 8);
    const size_t o_slow = plan.add(slots * 4), o_nslow = plan.add(4);
    const size_t o_draws = plan.add((size_t)n * draw_stride_full * 4);
    const size_t n_tab = coded ? coded->idx.size() : 0;
    const size_t o_cidx = plan.add(n_tab * 4 + 4), o_cfrac = plan.add(n_tab * 8 + 8);
    unsigned char *blk = arena_block(ctx, plan.total);
    if (!blk) { rc = 2; break; }
    unsigned *count_a = (unsigned *)(blk + o_ca), *off_a = (unsigned *)(blk + o_oa);
    unsigned *count_b = (unsigned *)(blk + o_cb), *off_b = (unsigned *)(blk + o_ob);
    unsigned *total_a = (unsigned *)(blk + o_ta), *total_ab = (unsigned *)(blk + o_tab);
    unsigned char *selected = blk + o_sel;
    double *nuttall = (double *)(blk + o_nut);
    unsigned *draws = (unsigned *)(blk + o_draws);
    dev_memcpy_h2d(ctx, nuttall, nuttall_host, (size_t)p.win_len * 8);
    const double *f0 = b.f0 + (size_t)u0 * b.f_stride;
    const int *f_len = b.f_len + u0;
    p.x = b.x + (size_t)u0 * b.x_stride; p.x_len = b.x_len + u0; p.x_stride = b.x_stride;
    p.time_axis = b.time_axis + (size_t)u0 * b.f_stride; p.f0 = f0; p.f_len = f_len;
    p.f_stride = b.f_stride;
    p.nuttall = nuttall; p.draws = draws; p.draw_stride = draw_stride_full;
    p.off_a = off_a; p.count_b = count_b; p.off_b = off_b; p.selected = selected;
    p.out = aperiodicity ? aperiodicity + (size_t)u0 * b.f_stride * bins : nullptr;
    p.tw = ctx->twiddle; p.status = ctx->status_dev;
    p.tw_body = ctx->twiddle_sized + tw_sized_offset(p.d_lg);
    if (coded) {
      rc = dev_memcpy_h2d(ctx, blk + o_cidx, coded->idx.data(), n_tab * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_cfrac, coded->frac.data(), n_tab * 8);
      if (rc) break;
      p.c_n = coded->dims; p.c_idx = (const int *)(blk + o_cidx); p.c_frac = (const double *)(blk + o_cfrac);
      p.c_out = coded_out + (size_t)u0 * b.f_stride * coded->dims;
    }
    p.slow_list = (int *)(blk + o_slow); p.slow_count = (int *)(blk + o_nslow);
    dev_memset(ctx, p.slow_count, 0, 4);

    WB_LAUNCH_FLAT(d4c_count_a_kernel, dim3((unsigned)((slots + 255) / 256)), 256, 0, ctx->stream, f0,
                   f_len, b.f_stride, n, fs, count_a);
    scan_counts(ctx, count_a, f_len, b.f_stride, nullptr, off_a, total_a, n);
    rng_fill(ctx, total_a, draws, draw_stride_full, max_a * (size_t)b.max_f_len, n);
    WB_LAUNCH_COOP(d4c_lovetrain_kernel, dim3((unsigned)b.max_f_len, (unsigned)n), lt_threads, smem_lt,
                   ctx->stream, p);
    scan_counts(ctx, count_b, f_len, b.f_stride, total_a, off_b, total_ab, n);
    // regenerates the pass-A prefix as well (identical values) -- simple, and pass A is ~20 % of the stream
    rng_fill(ctx, total_ab, draws, draw_stride_full, draw_stride_full, n);
    if (all_slow)
      WB_LAUNCH_FLAT(d4c_list_all_kernel, dim3((unsigned)((slots + 255) / 256)), 256, 0, ctx->stream, p, n);
    else
      WB_LAUNCH_COOP(d4c_body_kernel, dim3((unsigned)b.max_f_len, (unsigned)n), body_threads, smem_body,
                     ctx->stream, p);
    // long windows (f0 near the floor): persistent CTAs over the list the fast kernel filled, usually empty
    WB_LAUNCH_COOP(d4c_body_slow_kernel, dim3((unsigned)(2 * ctx->sm_count)), slow_threads, smem_slow, ctx->stream, p);
    rc = dev_check(ctx, "d4c");
  }
  // nuttall_host was copied with an async copy from pageable memory: the runtime stages it
  // before returning, so it can be released here.
  delete[] nuttall_host;
  return rc;
}

}  // namespace wb
