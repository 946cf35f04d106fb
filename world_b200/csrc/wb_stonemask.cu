// wb_stonemask.cu -- K-SM: F0 refinement by instantaneous frequency, one CTA per frame.
//
// Replaces StoneMask() (stonemask.cpp:212-218) and GetRefinedF0/GetMeanF0/GetSpectra/FixF0
// (:24-208).  Algorithm card: SURVEY.md A4.  The reference builds an FFT plan per frame and
// runs two full FFTs of 2^(2+floor(log2(2h+1))) points, but FixF0 only ever reads <= 2 + 6 bins
// of each spectrum; here those bins are evaluated directly (sparse DFT over the 2h+1 windowed
// samples with exact table twiddles), which is the same linear functional of the data.
#include "wb_internal.h"

namespace wb {

struct SmParams {
  const double *x; const int *x_len; int x_stride;
  const double *time_axis; const double *f0; const int *f_len; int f_stride;
  int fs; double *out; const double2 *tw;
  // packed inputs: utterance u's samples at x + x_off[u], its frames (inputs and output) at f_off[u] + i; null: padded
  const long long *x_off, *f_off;
};

// exp(-j 2 pi idx / WB_TW_N) for idx in [0, WB_TW_N)
WB_DEV double2 tw_full(const double2 *__restrict__ tw, int idx) {
  double2 w = __ldg(&tw[idx & (WB_TW_N / 2 - 1)]);
  if (idx & (WB_TW_N / 2)) { w.x = -w.x; w.y = -w.y; }
  return w;
}

WB_DEV double sm_window(double t, int raw_index, int fs, double T) {
  const double tmp = (raw_index - 1.0) / fs - t;
  return 0.42 + 0.5 * cos(2.0 * kPi * tmp / T) + 0.08 * cos(4.0 * kPi * tmp / T);
}

// FixF0 (stonemask.cpp:96-118) over the block: bins of `f_init`'s first H harmonics.
template <int H>
WB_DEV double sm_fix_f0(const double *xw, const double *xd, int nwin, int nfft, int lg_nfft, int fs,
                        double f_init, const double2 *__restrict__ tw, double *red) {
  const int tid = WB_TID, nth = WB_NTH;
  int bin[H];
#pragma unroll
  for (int m = 0; m < H; ++m)
    bin[m] = imin(round_half_away(f_init * nfft / fs * (m + 1)), nfft / 2);
  double acc[H][4];
#pragma unroll
  for (int m = 0; m < H; ++m) acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = 0.0;
  const int shift = WB_TW_LOG2 - lg_nfft;
  for (int j = tid; j < nwin; j += nth) {
    const double a = xw[j], d = xd[j];
#pragma unroll
    for (int m = 0; m < H; ++m) {
      const int idx = ((bin[m] * j) & (nfft - 1)) << shift;
      const double2 w = tw_full(tw, idx);
      acc[m][0] = fma(a, w.x, acc[m][0]);
      acc[m][1] = fma(a, w.y, acc[m][1]);
      acc[m][2] = fma(d, w.x, acc[m][2]);
      acc[m][3] = fma(d, w.y, acc[m][3]);
    }
  }
  double numerator = 0.0, denominator = 0.0;
#pragma unroll
  for (int m = 0; m < H; ++m) {
    block_sum_n<4>(acc[m], red);
    const double mr = acc[m][0], mi = acc[m][1], dr = acc[m][2], di = acc[m][3];
    const double num = mr * di - mi * dr;
    const double pw = mr * mr + mi * mi;
    const double inst = pw == 0.0 ? 0.0 : static_cast<double>(bin[m]) * fs / nfft + num / pw * fs / 2.0 / kPi;
    const double amp = sqrt(pw);
    numerator += amp * inst;
    denominator += amp * (m + 1);
  }
  return numerator / (denominator + kTiny);
}

WB_KERNEL(64, 8) stonemask_kernel(SmParams p) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const int u = blockIdx.y, i = blockIdx.x;
  if (i >= p.f_len[u]) return;
  const size_t fidx = p.x_off ? (size_t)(p.f_off[u] + i) : (size_t)u * p.f_stride + i;
  const double f0 = p.f0[fidx];
  const int fs = p.fs;
  if (f0 <= 40.0 || f0 > fs / 12.0) {  // kFloorF0StoneMask, stonemask.cpp:187-188
    if (tid == 0) p.out[fidx] = 0.0;
    return;
  }
  const double t = p.time_axis[fidx];
  const int h = static_cast<int>(1.5 * fs / f0 + 1.0);
  const int nwin = 2 * h + 1;
  int lg = 0;
  while ((2 << lg) <= nwin) ++lg;  // floor(log2(nwin)); nwin is odd so log()/kLog2 cannot sit on an integer
  const int lg_nfft = lg + 2, nfft = 1 << lg_nfft;
  const double T = (2.0 * h + 1.0) / fs;
  double *xw = smem, *xd = smem + nwin, *red = xd + nwin;
  const double *x = p.x_off ? p.x + p.x_off[u] : p.x + (size_t)u * p.x_stride;
  const int x_len = p.x_len[u];
  for (int j = tid; j < nwin; j += nth) {
    // index_raw[j] = round((t + base_time[j]) * fs), base_time[j] = (j - h) / fs  (:24-28, :193-194)
    const int r0 = round_half_away((t + static_cast<double>(j - h) / fs) * fs);
    const double w0 = sm_window(t, r0, fs, T);
    double dw;
    if (j == 0) {
      const int r1 = round_half_away((t + static_cast<double>(j + 1 - h) / fs) * fs);
      dw = -sm_window(t, r1, fs, T) / 2.0;
    } else if (j == nwin - 1) {
      const int rm = round_half_away((t + static_cast<double>(j - 1 - h) / fs) * fs);
      dw = sm_window(t, rm, fs, T) / 2.0;
    } else {
      const int r1 = round_half_away((t + static_cast<double>(j + 1 - h) / fs) * fs);
      const int rm = round_half_away((t + static_cast<double>(j - 1 - h) / fs) * fs);
      dw = -(sm_window(t, r1, fs, T) - sm_window(t, rm, fs, T)) / 2.0;
    }
    const double s = x[imax(0, imin(x_len - 1, r0 - 1))];
    xw[j] = s * w0;
    xd[j] = s * dw;
  }
  WB_SYNC();
  double mean_f0 = 0.0;
  const double tentative = sm_fix_f0<2>(xw, xd, nwin, nfft, lg_nfft, fs, f0, p.tw, red);
  if (!(tentative <= 0.0 || tentative > f0 * 2)) mean_f0 = sm_fix_f0<6>(xw, xd, nwin, nfft, lg_nfft, fs, tentative, p.tw, red);
  if (fabs(mean_f0 - f0) > f0 * 0.2) mean_f0 = f0;
  if (tid == 0) p.out[fidx] = mean_f0;
}

// the longest window (f0 at 40 Hz) of the kernel's transforms
static int sm_nwin_max(int fs) { return 2 * static_cast<int>(1.5 * fs / 40.0 + 1.0) + 1; }

bool stonemask_fits(int fs) {
  int lg = 0;
  while ((2 << lg) <= sm_nwin_max(fs)) ++lg;
  return (1 << (lg + 2)) <= WB_TW_N;
}

int stonemask_run(Ctx *ctx, const Batch &b, double *refined_f0) {
  if (b.n <= 0 || b.max_f_len <= 0) return 0;
  const int nwin_max = sm_nwin_max(b.fs);
  const size_t smem = (size_t)(2 * nwin_max + WB_REDN_DOUBLES) * sizeof(double);
#ifndef WB_EMU
  cudaFuncSetAttribute(stonemask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  SmParams p;
  p.x = b.x; p.x_len = b.x_len; p.x_stride = b.x_stride; p.time_axis = b.time_axis; p.f0 = b.f0;
  p.f_len = b.f_len; p.f_stride = b.f_stride; p.fs = b.fs; p.out = refined_f0; p.tw = ctx->twiddle;
  p.x_off = b.x_off; p.f_off = b.f_off;
  if (b.x_off) {   // packed inputs: the packed stage call's chunks have at most 65535 utterances
    WB_LAUNCH_COOP(stonemask_kernel, dim3((unsigned)b.max_f_len, (unsigned)b.n), 64, smem, ctx->stream, p);
    return dev_check(ctx, "stonemask");
  }
  for (int u0 = 0; u0 < b.n; u0 += 65535) {
    const int n = imin(65535, b.n - u0);
    SmParams q = p;
    q.x += (size_t)u0 * b.x_stride; q.x_len += u0; q.time_axis += (size_t)u0 * b.f_stride;
    q.f0 += (size_t)u0 * b.f_stride; q.f_len += u0; q.out += (size_t)u0 * b.f_stride;
    WB_LAUNCH_COOP(stonemask_kernel, dim3((unsigned)b.max_f_len, (unsigned)n), 64, smem, ctx->stream, q);
  }
  return dev_check(ctx, "stonemask");
}

}  // namespace wb
