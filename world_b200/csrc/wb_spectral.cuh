// wb_spectral.cuh -- block-cooperative restatements of the reference's shared spectral
// helpers (SURVEY.md A0): DCCorrection (common.cpp:56-75), LinearSmoothing (common.cpp:27-46,
// 77-111), interp1Q (matlabfunctions.cpp:214-235), and the draw -> normal mapping of randn
// (matlabfunctions.cpp:263).  All operate on shared-memory vectors of fft_size/2+1 doubles.
#pragma once
#include "wb_platform.cuh"
#include "wb_block.cuh"

namespace wb {

// randn(): tmp / 268435456.0 - 6.0 with tmp the stored 32-bit sum
WB_DEV double randn_value(unsigned tmp) { return (double)tmp / 268435456.0 - 6.0; }

// cos(theta) for |theta| <= ~4 (window arguments: never beyond pi (1 + 1/(2h+1)) for f0 the estimators produce,
// pi 7/6 for a caller-supplied f0 at fs/2): cos = 1 - 2 sin^2(theta/2), sin by its Taylor series to x^25
// (|x| <= 2: truncation < 2e-20).  ~16 FP64 operations instead of the ~45 of the general-purpose cos(); ~2 ulp.
WB_DEV double cos_small(double theta) {
  const double x = 0.5 * theta, x2 = x * x;
  double p = -1.0 / 15511210043330985984000000.0;             // -1/25!
  p = fma(p, x2, 1.0 / 25852016738884976640000.0);            // +1/23!
  p = fma(p, x2, -1.0 / 51090942171709440000.0);              // -1/21!
  p = fma(p, x2, 1.0 / 121645100408832000.0);                 // +1/19!
  p = fma(p, x2, -1.0 / 355687428096000.0);                   // -1/17!
  p = fma(p, x2, 1.0 / 1307674368000.0);                      // +1/15!
  p = fma(p, x2, -1.0 / 6227020800.0);                        // -1/13!
  p = fma(p, x2, 1.0 / 39916800.0);                           // +1/11!
  p = fma(p, x2, -1.0 / 362880.0);                            // -1/9!
  p = fma(p, x2, 1.0 / 5040.0);                               // +1/7!
  p = fma(p, x2, -1.0 / 120.0);                               // -1/5!
  p = fma(p, x2, 1.0 / 6.0);                                  // +1/3!  (sign folded below)
  const double sn = x - x * x2 * p;                           // sin(x) = x - x^3/3! + x^5/5! - ...
  return 1.0 - 2.0 * sn * sn;
}

// One interp1Q sample: y[base] + (y[base+1]-y[base]) * frac with base = int((xi-x0)/dx); the caller passes 1/dx
// (the quotient only positions a linear interpolation: a last-digit difference moves the result continuously, also
// across an integer).  The reference zeroes delta_y[ny-1]; `ny` reproduces that.
// kExact: divide by dx like the reference (CheapTrick: its output bins are differences of two interpolated running
// sums, and bins 120 dB below the peak see every last digit -- App. B4); otherwise multiply by the reciprocal.
template <bool kExact>
WB_DEV double interp1q_at(double x0, double dx, double inv_dx, const double *y, int ny, double xi) {
  const double r = kExact ? (xi - x0) / dx : (xi - x0) * inv_dx;
  const int base = static_cast<int>(r);
  const double frac = r - base;
  const double dy = (base + 1 < ny) ? (y[base + 1] - y[base]) : 0.0;
  return y[base] + dy * frac;
}

// DCCorrection(in -> in, in place).  `tmp` needs upper_limit doubles.  Ends with a barrier.
template <bool kExact = false>
WB_DEV void dc_correction(double *spec, double f0, int fs, int fft_size, double *tmp) {
  const int tid = WB_TID, nth = WB_NTH;
  // f0 is caller supplied: at or above fs/2 (or non-finite) the reference indexes past its arrays.  Here such a
  // value is clamped two bins below the Nyquist bin -- every index stays inside the fft_size/2 + 1 values of
  // `spec`; the row is meaningless either way, but there is no fault.  The reference stays in bounds up to one bin
  // below Nyquist, so between two and one bin below it the clamp would move the interpolation's origin -- but no such
  // row is kept: both callers' linear_smoothing then refuses the frame (status 2), as it does every f0 above 3/8 fs
  // (CheapTrick) or fs/4 (D4C).
  f0 = dmin(dmax(f0, 0.0), (0.5 - 2.0 / fft_size) * fs);
  const int upper_limit = 2 + static_cast<int>(f0 * fft_size / fs);
  const int n_rep = upper_limit - 1;
  const double dx = -static_cast<double>(fs) / fft_size, inv_dx = -static_cast<double>(fft_size) / fs;
  const double inv_n = 1.0 / fft_size;          // exact: fft_size is a power of two
  WB_UNROLL4
  for (int i = tid; i < n_rep; i += nth) {
    const double xi = static_cast<double>(i) * fs * inv_n;
    tmp[i] = interp1q_at<kExact>(f0, dx, inv_dx, spec, upper_limit + 1, xi);
  }
  WB_SYNC();
  WB_UNROLL4
  for (int i = tid; i < n_rep; i += nth) spec[i] = spec[i] + tmp[i];
  WB_SYNC();
}

// Capacity (in doubles) the `seg` scratch of linear_smoothing must have for a given half size.
WB_HD inline int smoothing_capacity(int fft_size) { return fft_size + 2; }

// LinearSmoothing(in -> out); in == out allowed.  `seg` is scratch of smoothing_capacity().
// kSequential = true reproduces the reference's index-order running sum bit for bit
// (mandatory for CheapTrick, SURVEY.md App. B4); false uses a blocked scan (D4C: measured
// insensitive).  Returns false (all threads) if the smoothing width does not fit the scratch.
template <bool kSequential>
WB_DEV bool linear_smoothing(const double *in, double width, int fs, int fft_size, double *out,
                             double *seg, double *red_big) {
  const int tid = WB_TID, nth = WB_NTH;
  const int half = fft_size / 2;
  // a caller-supplied f0 makes the width anything, infinite included: it is tested before the conversion to int
  // (boundary > half exactly when width * fft_size / fs >= half), which would otherwise wrap round into range
  const double b = width * fft_size / fs;
  if (!(b < half)) return false;
  const int boundary = static_cast<int>(b) + 1;
  const int n_ext = half + boundary * 2 + 1;
  if (n_ext > smoothing_capacity(fft_size)) return false;

  const double inv_n = 1.0 / fft_size;          // exact: fft_size is a power of two
  // mirror-extend and scale:  seg[i] = ext[i] * fs / fft_size   (common.cpp:30-41)
  WB_UNROLL4
  for (int i = tid; i < n_ext; i += nth) {
    double v;
    if (i < boundary) v = in[boundary - i];
    else if (i < half + boundary) v = in[i - boundary];
    else v = in[half - (i - (half + boundary))];
    seg[i] = v * fs * inv_n;   // == v * fs / fft_size bit for bit (power of two)
  }
  WB_SYNC();
  if (kSequential) {
    if (tid == 0) {
      // index-order running sum: eight loads in flight, then eight dependent adds (the chain is the
      // DADD latency, not load + add + store per element)
      double run = seg[0];
      int i = 1;
      for (; i + 8 <= n_ext; i += 8) {
        double v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = seg[i + k];
#pragma unroll
        for (int k = 0; k < 8; ++k) { run = v[k] + run; v[k] = run; }
#pragma unroll
        for (int k = 0; k < 8; ++k) seg[i + k] = v[k];
      }
      for (; i < n_ext; ++i) { run = seg[i] + run; seg[i] = run; }
    }
    WB_SYNC();
  } else {
    block_inclusive_scan(seg, n_ext, red_big);
  }
  const double origin = -(boundary - 0.5) * fs / fft_size;
  const double dx = static_cast<double>(fs) / fft_size, inv_dx = static_cast<double>(fft_size) / fs, inv_width = 1.0 / width;
  WB_UNROLL4
  for (int i = tid; i <= half; i += nth) {
    const double lo_x = static_cast<double>(i) * inv_n * fs - width / 2.0;
    const double hi_x = lo_x + width;
    const double lo = interp1q_at<kSequential>(origin, dx, inv_dx, seg, n_ext, lo_x);
    const double hi = interp1q_at<kSequential>(origin, dx, inv_dx, seg, n_ext, hi_x);
    out[i] = kSequential ? (hi - lo) / width : (hi - lo) * inv_width;
  }
  WB_SYNC();
  return true;
}

}  // namespace wb
