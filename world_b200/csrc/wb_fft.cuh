// wb_fft.cuh -- shared-memory FFTs for the frame kernels (FP64, power-of-two, forward only).
//
// Replaces the reference's L1 layer (src/fft.cpp, an Ooura split-radix FFT behind an
// FFTW-shaped plan API, fft.h:37-44) for every per-frame transform.  It is NOT a port of that
// code: transforms live entirely in shared memory, are executed cooperatively by one CTA, and
// only the conventions are kept (SURVEY.md App. A0):
//   r2c : X[k] = sum_n x[n] exp(-j 2 pi k n / N), k = 0..N/2          (fft.cpp:49-60)
//   c2r of a real, even spectrum == Re r2c(mirror(spectrum))           (fft.cpp:26-35)
// so every transform the analysis path needs is a forward real FFT.
//
// Twiddles come from one table tw[k] = exp(-j 2 pi k / WB_TW_N), k < WB_TW_N/2, computed on
// the host in long double and kept in global memory (L1/L2 resident, read with __ldg).
#pragma once
#include "wb_platform.cuh"

namespace wb {

#define WB_TW_LOG2 13
#define WB_TW_N (1 << WB_TW_LOG2)  // supports complex FFTs up to 8192, real up to 8192

WB_DEV unsigned bit_reverse(unsigned v, int bits) {
#ifdef WB_EMU
  unsigned r = 0;
  for (int i = 0; i < bits; ++i) { r = (r << 1) | (v & 1u); v >>= 1; }
  return r;
#else
  return __brev(v) >> (32 - bits);
#endif
}

WB_DEV double2 cmul(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -(a.y * b.y)), fma(a.x, b.y, a.y * b.x));
}
WB_DEV double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
WB_DEV double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
WB_DEV double2 mul_mj(double2 a) { return make_double2(a.y, -a.x); }  // (-j) * a

// DIT stages s, s+1 as one radix-4 pass (quarter = 2^(s-1)); one table twiddle, the other is its square.
WB_DEV void fft_pass_radix4(double2 *z, int n, int s, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int quarter = 1 << (s - 1);
  const int tws = WB_TW_LOG2 - (s + 1);
  for (int q = tid; q < (n >> 2); q += nth) {
    const int j = q & (quarter - 1);
    const int i0 = ((q >> (s - 1)) << (s + 1)) + j;
    const int i1 = i0 + quarter, i2 = i1 + quarter, i3 = i2 + quarter;
    const double2 b = __ldg(&tw[j << tws]);  // exp(-j 2 pi j / (4 quarter))
    const double2 a = cmul(b, b);
    const double2 z0 = z[i0], z1 = z[i1], z2 = z[i2], z3 = z[i3];
    const double2 t1 = cmul(a, z1), t3 = cmul(a, z3);
    const double2 u0 = cadd(z0, t1), u1 = csub(z0, t1), u2 = cadd(z2, t3), u3 = csub(z2, t3);
    const double2 v2 = cmul(b, u2), w3 = mul_mj(cmul(b, u3));
    z[i0] = cadd(u0, v2); z[i2] = csub(u0, v2);
    z[i1] = cadd(u1, w3); z[i3] = csub(u1, w3);
  }
  WB_SYNC();
}

// DIT stages s, s+1, s+2 as one radix-8 pass held in registers (q = 2^(s-1), elements i0 + k q):
// a third of the shared-memory passes of radix-2.  One table twiddle c = W_{8q}^j; b = c^2, a = c^4;
// the remaining factors are the constants W_8^k.
WB_DEV void fft_pass_radix8(double2 *z, int n, int s, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int q = 1 << (s - 1);
  const int tws = WB_TW_LOG2 - (s + 2);
  const double r = 0.70710678118654752440;
  for (int t = tid; t < (n >> 3); t += nth) {
    const int j = t & (q - 1);
    const int i0 = ((t >> (s - 1)) << (s + 2)) + j;
    const double2 c = __ldg(&tw[j << tws]);
    const double2 b = cmul(c, c);
    const double2 a = cmul(b, b);
    double2 x0 = z[i0], x1 = z[i0 + q], x2 = z[i0 + 2 * q], x3 = z[i0 + 3 * q];
    double2 x4 = z[i0 + 4 * q], x5 = z[i0 + 5 * q], x6 = z[i0 + 6 * q], x7 = z[i0 + 7 * q];
    // stage s: (0,1) (2,3) (4,5) (6,7), twiddle a
    double2 t1 = cmul(a, x1), t3 = cmul(a, x3), t5 = cmul(a, x5), t7 = cmul(a, x7);
    const double2 y0 = cadd(x0, t1), y1 = csub(x0, t1), y2 = cadd(x2, t3), y3 = csub(x2, t3);
    const double2 y4 = cadd(x4, t5), y5 = csub(x4, t5), y6 = cadd(x6, t7), y7 = csub(x6, t7);
    // stage s+1: (0,2) (4,6) twiddle b; (1,3) (5,7) twiddle -j b
    const double2 u2 = cmul(b, y2), u6 = cmul(b, y6), u3 = mul_mj(cmul(b, y3)), u7 = mul_mj(cmul(b, y7));
    const double2 w0 = cadd(y0, u2), w2 = csub(y0, u2), w1 = cadd(y1, u3), w3 = csub(y1, u3);
    const double2 w4 = cadd(y4, u6), w6 = csub(y4, u6), w5 = cadd(y5, u7), w7 = csub(y5, u7);
    // stage s+2: (k, k+4) twiddle c W_8^k
    const double2 v4 = cmul(c, w4);
    const double2 c5 = cmul(c, w5), v5 = make_double2((c5.x + c5.y) * r, (c5.y - c5.x) * r);
    const double2 v6 = mul_mj(cmul(c, w6));
    const double2 c7 = cmul(c, w7), v7 = make_double2((c7.y - c7.x) * r, -(c7.x + c7.y) * r);
    z[i0] = cadd(w0, v4);         z[i0 + 4 * q] = csub(w0, v4);
    z[i0 + q] = cadd(w1, v5);     z[i0 + 5 * q] = csub(w1, v5);
    z[i0 + 2 * q] = cadd(w2, v6); z[i0 + 6 * q] = csub(w2, v6);
    z[i0 + 3 * q] = cadd(w3, v7); z[i0 + 7 * q] = csub(w3, v7);
  }
  WB_SYNC();
}

WB_DEV void fft_pass_radix2(double2 *z, int n, int s, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int half = 1 << (s - 1);
  const int tws = WB_TW_LOG2 - s;
  for (int b = tid; b < (n >> 1); b += nth) {
    const int j = b & (half - 1);
    const int i0 = ((b >> (s - 1)) << s) + j;
    const double2 w = __ldg(&tw[j << tws]);
    const double2 u = z[i0], v = cmul(w, z[i0 + half]);
    z[i0] = cadd(u, v);
    z[i0 + half] = csub(u, v);
  }
  WB_SYNC();
}

// In-place forward complex FFT of z[0..2^lg) (natural order in, natural order out).
// Bit reversal, then decimation-in-time stages grouped into radix-8 passes held in registers (plus
// one or two radix-4 passes, or a radix-2 pass for lg < 2, to make the stage count come out):
// lg = 9 (CheapTrick) takes 3 passes, lg = 10 / 11 (D4C) take 4.  Ends with a barrier.
WB_DEV void cfft_forward(double2 *z, int lg, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int n = 1 << lg;
  for (int i = tid; i < n; i += nth) {
    const int j = (int)bit_reverse((unsigned)i, lg);
    if (i < j) { const double2 a = z[i]; z[i] = z[j]; z[j] = a; }
  }
  WB_SYNC();
  int s = 1;
  if (lg == 1) { fft_pass_radix2(z, n, 1, tw); return; }
  // number of radix-4 passes so that the rest is a multiple of three stages
  int n4 = (lg % 3 == 0) ? 0 : ((lg % 3 == 2) ? 1 : 2);
  if (lg < 4 && lg % 3 == 1) n4 = lg / 2;  // lg = 1 handled above; (lg = 4 -> two radix-4 passes)
  for (int k = 0; k < n4; ++k, s += 2) fft_pass_radix4(z, n, s, tw);
  for (; s + 2 <= lg; s += 3) fft_pass_radix8(z, n, s, tw);
}

// Forward real FFT of buf[0..N), N = 2^lg >= 4, in place: on return buf holds N/2+1 complex
// values (buf must have room for N+2 doubles).  Ends with a barrier.
WB_DEV void rfft_forward(double *buf, int lg, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  double2 *z = reinterpret_cast<double2 *>(buf);
  const int m = 1 << (lg - 1);
  cfft_forward(z, lg - 1, tw);
  const int tws = WB_TW_LOG2 - lg;
  WB_UNROLL4
  for (int k = tid; k <= (m >> 1); k += nth) {
    if (k == 0) {
      const double2 z0 = z[0];
      z[0] = make_double2(z0.x + z0.y, 0.0);
      z[m] = make_double2(z0.x - z0.y, 0.0);
    } else {
      const double2 a = z[k], b = z[m - k];
      const double er = 0.5 * (a.x + b.x), ei = 0.5 * (a.y - b.y);
      const double orr = 0.5 * (a.y + b.y), oi = -0.5 * (a.x - b.x);
      const double2 w = __ldg(&tw[k << tws]);
      const double pr = fma(w.x, orr, -(w.y * oi));
      const double pi = fma(w.x, oi, w.y * orr);
      z[k] = make_double2(er + pr, ei + pi);
      z[m - k] = make_double2(er - pr, -(ei - pi));
    }
  }
  WB_SYNC();
}

// Two real FFTs from one complex FFT: z[n] = a[n] + j b[n] has been transformed in place by
// cfft_forward (size n = 2^lg); returns A[k] and B[k] for 0 <= k <= n/2.
WB_DEV void split_pair(const double2 *z, int n, int k, double2 &A, double2 &B) {
  const double2 p = z[k], q = z[(n - k) & (n - 1)];
  A = make_double2(0.5 * (p.x + q.x), 0.5 * (p.y - q.y));
  B = make_double2(0.5 * (p.y + q.y), -0.5 * (p.x - q.x));
}

// =============================================================================================
// Stockham (self-sorting) FFT, round 2.  The in-place DIT above needs a bit-reversal pass and its first
// passes walk shared memory with power-of-two strides of double2: a large share of the shared wavefronts of
// the frame kernels were bank conflicts.  The transform below goes natural order in ->
// natural order out with NO permutation pass, ping-ponging between two buffers (one barrier per pass, any
// block size, also one emulated thread), and every access is conflict free:
//   * layout: element i of a buffer lives at fpad(i) = i + (i >> 3) (one spare double2 per 8);
//   * reads  x[i + r T] (T = n / R): eight consecutive threads read eight consecutive double2;
//   * writes y[j + m p], j = (i - k) R + k, k = i & (p - 1): for p >= 8 again consecutive; for p = 1, 2, 4 the
//     stride-R pattern lands on distinct 16-byte bank groups because of the padding.
// Pass structure (DIT Stockham): p = product of the radices already applied; thread i loads u[r] = x[i + r T],
// multiplies by w^r, w = exp(-j 2 pi k / (p R)), does an R-point DFT and stores y[j + m p].  The first pass
// has k = 0, i.e. no twiddles at all, so it is always the radix-8 one.  The radix-8 arithmetic is the
// register butterfly of fft_pass_radix8 (three DIT stages with twiddles w^4, w^2, w).
WB_DEV int fpad(int i) { return i + (i >> 3); }
// double2 slots a padded buffer of n complex values needs
#define WB_FPAD_SLOTS(n) ((n) + ((n) >> 3) + 1)
// index, in doubles, of real sample e of a sequence packed two per complex slot (z[e >> 1].{x, y})
WB_DEV int rpad(int e) { return (fpad(e >> 1) << 1) | (e & 1); }

// x[]: inputs in bit-reversed slot order (x[bitrev3(r)] = u[r]); on return x[m] = sum_r u[r] w^r W_8^{r m}
template <bool kTw>
WB_DEV void radix8_butterfly(double2 (&x)[8], double2 c) {
  const double r = 0.70710678118654752440;
  double2 y0, y1, y2, y3, y4, y5, y6, y7;
  if (kTw) {
    const double2 b = cmul(c, c);
    const double2 a = cmul(b, b);
    const double2 t1 = cmul(a, x[1]), t3 = cmul(a, x[3]), t5 = cmul(a, x[5]), t7 = cmul(a, x[7]);
    y0 = cadd(x[0], t1); y1 = csub(x[0], t1); y2 = cadd(x[2], t3); y3 = csub(x[2], t3);
    y4 = cadd(x[4], t5); y5 = csub(x[4], t5); y6 = cadd(x[6], t7); y7 = csub(x[6], t7);
    const double2 u2 = cmul(b, y2), u6 = cmul(b, y6), u3 = mul_mj(cmul(b, y3)), u7 = mul_mj(cmul(b, y7));
    const double2 w0 = cadd(y0, u2), w2 = csub(y0, u2), w1 = cadd(y1, u3), w3 = csub(y1, u3);
    const double2 w4 = cadd(y4, u6), w6 = csub(y4, u6), w5 = cadd(y5, u7), w7 = csub(y5, u7);
    const double2 v4 = cmul(c, w4);
    const double2 c5 = cmul(c, w5), v5 = make_double2((c5.x + c5.y) * r, (c5.y - c5.x) * r);
    const double2 v6 = mul_mj(cmul(c, w6));
    const double2 c7 = cmul(c, w7), v7 = make_double2((c7.y - c7.x) * r, -(c7.x + c7.y) * r);
    x[0] = cadd(w0, v4); x[4] = csub(w0, v4); x[1] = cadd(w1, v5); x[5] = csub(w1, v5);
    x[2] = cadd(w2, v6); x[6] = csub(w2, v6); x[3] = cadd(w3, v7); x[7] = csub(w3, v7);
  } else {
    y0 = cadd(x[0], x[1]); y1 = csub(x[0], x[1]); y2 = cadd(x[2], x[3]); y3 = csub(x[2], x[3]);
    y4 = cadd(x[4], x[5]); y5 = csub(x[4], x[5]); y6 = cadd(x[6], x[7]); y7 = csub(x[6], x[7]);
    const double2 u3 = mul_mj(y3), u7 = mul_mj(y7);
    const double2 w0 = cadd(y0, y2), w2 = csub(y0, y2), w1 = cadd(y1, u3), w3 = csub(y1, u3);
    const double2 w4 = cadd(y4, y6), w6 = csub(y4, y6), w5 = cadd(y5, u7), w7 = csub(y5, u7);
    const double2 v5 = make_double2((w5.x + w5.y) * r, (w5.y - w5.x) * r);
    const double2 v6 = mul_mj(w6);
    const double2 v7 = make_double2((w7.y - w7.x) * r, -(w7.x + w7.y) * r);
    x[0] = cadd(w0, w4); x[4] = csub(w0, w4); x[1] = cadd(w1, v5); x[5] = csub(w1, v5);
    x[2] = cadd(w2, v6); x[6] = csub(w2, v6); x[3] = cadd(w3, v7); x[7] = csub(w3, v7);
  }
}

template <bool kTw>
WB_DEV void sfft_pass8(const double2 *src, double2 *dst, int n, int lgp, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int T = n >> 3, p = 1 << lgp;
  for (int i = tid; i < T; i += nth) {
    const int k = i & (p - 1), j = ((i - k) << 3) + k;
    double2 x[8];
    x[0] = src[fpad(i)];         x[4] = src[fpad(i + T)];     x[2] = src[fpad(i + 2 * T)]; x[6] = src[fpad(i + 3 * T)];
    x[1] = src[fpad(i + 4 * T)]; x[5] = src[fpad(i + 5 * T)]; x[3] = src[fpad(i + 6 * T)]; x[7] = src[fpad(i + 7 * T)];
    double2 c = make_double2(1.0, 0.0);
    if (kTw) c = __ldg(&tw[k << (WB_TW_LOG2 - lgp - 3)]);
    radix8_butterfly<kTw>(x, c);
#pragma unroll
    for (int m = 0; m < 8; ++m) dst[fpad(j + m * p)] = x[m];
  }
  WB_SYNC();
}

WB_DEV void sfft_pass4(const double2 *src, double2 *dst, int n, int lgp, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int T = n >> 2, p = 1 << lgp;
  for (int i = tid; i < T; i += nth) {
    const int k = i & (p - 1), j = ((i - k) << 2) + k;
    const double2 u0 = src[fpad(i)], u1 = src[fpad(i + T)], u2 = src[fpad(i + 2 * T)], u3 = src[fpad(i + 3 * T)];
    const double2 b = __ldg(&tw[k << (WB_TW_LOG2 - lgp - 2)]);
    const double2 a = cmul(b, b);
    const double2 t2 = cmul(a, u2), t3 = cmul(a, u3);
    const double2 y0 = cadd(u0, t2), y1 = csub(u0, t2), y2 = cadd(u1, t3), y3 = csub(u1, t3);
    const double2 v2 = cmul(b, y2), v3 = mul_mj(cmul(b, y3));
    dst[fpad(j)] = cadd(y0, v2);         dst[fpad(j + 2 * p)] = csub(y0, v2);
    dst[fpad(j + p)] = cadd(y1, v3);     dst[fpad(j + 3 * p)] = csub(y1, v3);
  }
  WB_SYNC();
}

WB_DEV void sfft_pass2(const double2 *src, double2 *dst, int n, int lgp, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH;
  const int T = n >> 1, p = 1 << lgp;
  for (int i = tid; i < T; i += nth) {
    const int k = i & (p - 1), j = ((i - k) << 1) + k;
    const double2 u0 = src[fpad(i)];
    const double2 v = cmul(__ldg(&tw[k << (WB_TW_LOG2 - lgp - 1)]), src[fpad(i + T)]);
    dst[fpad(j)] = cadd(u0, v);
    dst[fpad(j + p)] = csub(u0, v);
  }
  WB_SYNC();
}

// Forward complex FFT of the 2^lg values in padded buffer `a` (natural order); `b` is a second padded buffer of
// the same size.  Both are clobbered; returns the one that holds the result (natural order, padded).  The caller
// must have made `a` visible (barrier) before the call; ends with a barrier.
WB_DEV double2 *sfft_forward(double2 *a, double2 *b, int lg, const double2 *__restrict__ tw) {
  const int n = 1 << lg;
  double2 *src = a, *dst = b;
  int lgp = 0;
  if (lg >= 3) {
    sfft_pass8<false>(src, dst, n, 0, tw);
    double2 *t = src; src = dst; dst = t;
    lgp = 3;
    for (; lg - lgp >= 3; lgp += 3) {
      sfft_pass8<true>(src, dst, n, lgp, tw);
      t = src; src = dst; dst = t;
    }
  }
  if (lg - lgp == 2) {
    sfft_pass4(src, dst, n, lgp, tw);
    double2 *t = src; src = dst; dst = t;
  } else if (lg - lgp == 1) {
    sfft_pass2(src, dst, n, lgp, tw);
    double2 *t = src; src = dst; dst = t;
  }
  return src;
}

// Same transform in ONE padded buffer: every thread keeps the (at most) eight values it owns in a pass in
// registers -- load, barrier, butterflies + store, barrier.  Two barriers per pass instead of one, half the shared
// memory (more CTAs per SM for the barrier-heavy frame kernels).  Needs 2^lg <= 8 * blockDim.x.  Natural order in,
// natural order out, result in `a`; the caller must have made `a` visible; ends with a barrier.
WB_DEV_NOINLINE void sfft_forward_inplace(double2 *a, int lg, const double2 *__restrict__ tw) {
#ifdef WB_EMU
  // one emulated thread: run the ping-pong passes against a scratch buffer (same arithmetic), copy back
  static double2 tmp[WB_FPAD_SLOTS(WB_TW_N)];
  double2 *r = sfft_forward(a, tmp, lg, tw);
  if (r != a) for (int i = 0; i < WB_FPAD_SLOTS(1 << lg); ++i) a[i] = r[i];
#else
  const int tid = threadIdx.x, nth = blockDim.x;
  const int n = 1 << lg;
  int lgp = 0;
  if (lg >= 3) {
    const int T = n >> 3;
    for (; lg - lgp >= 3; lgp += 3) {
      const int p = 1 << lgp, i = tid;
      double2 x[8];
      if (i < T) {
        x[0] = a[fpad(i)];         x[4] = a[fpad(i + T)];     x[2] = a[fpad(i + 2 * T)]; x[6] = a[fpad(i + 3 * T)];
        x[1] = a[fpad(i + 4 * T)]; x[5] = a[fpad(i + 5 * T)]; x[3] = a[fpad(i + 6 * T)]; x[7] = a[fpad(i + 7 * T)];
      }
      __syncthreads();
      if (i < T) {
        const int k = i & (p - 1), j = ((i - k) << 3) + k;
        if (lgp == 0) {
          radix8_butterfly<false>(x, make_double2(1.0, 0.0));
        } else {
          radix8_butterfly<true>(x, __ldg(&tw[k << (WB_TW_LOG2 - lgp - 3)]));
        }
#pragma unroll
        for (int m = 0; m < 8; ++m) a[fpad(j + m * p)] = x[m];
      }
      __syncthreads();
    }
  }
  if (lg - lgp == 2) {
    const int T = n >> 2, p = 1 << lgp;
    double2 u[2][4];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = tid + q * nth;
      if (i < T) { u[q][0] = a[fpad(i)]; u[q][1] = a[fpad(i + T)]; u[q][2] = a[fpad(i + 2 * T)]; u[q][3] = a[fpad(i + 3 * T)]; }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = tid + q * nth;
      if (i < T) {
        const int k = i & (p - 1), j = ((i - k) << 2) + k;
        const double2 b = __ldg(&tw[k << (WB_TW_LOG2 - lgp - 2)]);
        const double2 aa = cmul(b, b);
        const double2 t2 = cmul(aa, u[q][2]), t3 = cmul(aa, u[q][3]);
        const double2 y0 = cadd(u[q][0], t2), y1 = csub(u[q][0], t2), y2 = cadd(u[q][1], t3), y3 = csub(u[q][1], t3);
        const double2 v2 = cmul(b, y2), v3 = mul_mj(cmul(b, y3));
        a[fpad(j)] = cadd(y0, v2);     a[fpad(j + 2 * p)] = csub(y0, v2);
        a[fpad(j + p)] = cadd(y1, v3); a[fpad(j + 3 * p)] = csub(y1, v3);
      }
    }
    __syncthreads();
  } else if (lg - lgp == 1) {
    const int T = n >> 1, p = 1 << lgp;
    double2 u[4][2];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = tid + q * nth;
      if (i < T) { u[q][0] = a[fpad(i)]; u[q][1] = a[fpad(i + T)]; }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = tid + q * nth;
      if (i < T) {
        const int k = i & (p - 1), j = ((i - k) << 1) + k;
        const double2 v = cmul(__ldg(&tw[k << (WB_TW_LOG2 - lgp - 1)]), u[q][1]);
        a[fpad(j)] = cadd(u[q][0], v);
        a[fpad(j + p)] = csub(u[q][0], v);
      }
    }
    __syncthreads();
  }
#endif
}

// Real FFT on top: the N = 2^lg real samples were packed two per slot (sample e at rpad(e)) and transformed as
// N/2 complex values by sfft_forward -> z.  Calls f(k, X[k]) once for every k in 0..N/2 (thread t handles k = t
// and N/2 - t), X = r2c of the real sequence.  No barrier; reads z only.
template <class F>
WB_DEV void rfft_unpack(const double2 *z, int lg, const double2 *__restrict__ tw, F f) {
  const int tid = WB_TID, nth = WB_NTH;
  const int m = 1 << (lg - 1);
  const int tws = WB_TW_LOG2 - lg;
  for (int k = tid; k <= (m >> 1); k += nth) {
    if (k == 0) {
      const double2 z0 = z[0];
      f(0, make_double2(z0.x + z0.y, 0.0));
      f(m, make_double2(z0.x - z0.y, 0.0));
    } else {
      const double2 a = z[fpad(k)], b = z[fpad(m - k)];
      const double er = 0.5 * (a.x + b.x), ei = 0.5 * (a.y - b.y);
      const double orr = 0.5 * (a.y + b.y), oi = -0.5 * (a.x - b.x);
      const double2 w = __ldg(&tw[k << tws]);
      const double pr = fma(w.x, orr, -(w.y * oi));
      const double pi = fma(w.x, oi, w.y * orr);
      f(k, make_double2(er + pr, ei + pi));
      if (k != m - k) f(m - k, make_double2(er - pr, -(ei - pi)));
    }
  }
}

}  // namespace wb
