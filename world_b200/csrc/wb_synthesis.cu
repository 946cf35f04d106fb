// wb_synthesis.cu -- batched WORLD synthesis (SURVEY.md 8 row f1: the first "next" component).
//
// Replaces Synthesis() (synthesis.cpp:339-399): time base and pulse placement (:223-326), per-pulse
// minimum-phase periodic response (:110-138) and aperiodic (noise) response (:36-69), overlap-add.
//   syn_timebase_kernel   utterance -> CTA: interp1 of f0 / vuv onto the sample grid, the
//                         index-order phase accumulation (its rounding decides where pulses fall,
//                         so it stays sequential on one thread), parallel wrap / pulse detection,
//                         ordered compaction, randn draw offsets
//   syn_pulse_kernel      (utterance, pulse) -> 128-thread CTA: envelope / aperiodicity interpolation,
//                         two GetMinimumPhaseSpectrum (common.cpp:192-226), noise spectrum, two
//                         inverse transforms, DC removal -> one response of fft_size samples; one launch
//                         per distinct fft_size of a pass, over the list of its utterances
//   syn_overlap_kernel    output sample -> thread: sums the responses covering it in pulse order
//                         (the reference's accumulation order, so the sum is deterministic)
// and, ahead of it, the voice modification of the reference demo (F0 scaling and formant shift, section below):
//   modify_stretch_kernel, modify_f0_kernel, and per frame modify_curve_stretch_kernel, modify_curve_f0_kernel
// FFT conventions (SURVEY.md App. A0): c2c FORWARD of a == FFT(conj a); c2r of X == Re FFT(conj X~)
// with X~ the Hermitian extension -- both are forward transforms of wb_fft.cuh.
#include "wb_chain.h"
#include "wb_spectral.cuh"
#include "../../include/world/matlabfunctions.h"
#include <algorithm>
#include <climits>
#include <map>
#include <stdio.h>
#include <type_traits>
#include <vector>

#ifdef WB_EMU
// the CUDA intrinsics the stretch uses; the emulation is compiled with -ffp-contract=off, so plain operators round
// each step on their own
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline void atomicMin(unsigned long long *p, unsigned long long v) { if (v < *p) *p = v; }
#endif

namespace wb {

struct SynParams {
  const double *f0; const int *f_len; int f_stride;
  const double *sp; const double *ap; int fft_size, lg_fft;
  int row;                  // doubles per sp / ap frame row (>= each utterance's fft_size / 2 + 1)
  const int *fft_u;         // [n] fft_size of each utterance, or null: fft_size for all
  const int *list;          // syn_pulse_kernel: the utterance of each blockIdx.y (all of size fft_size), or null
  double frame_period;      // seconds
  const double *fp_u;       // [n] frame period of each utterance (seconds), or null: frame_period for all
  int fs;
  const int *y_len; int y_stride;
  // time base scratch
  double *phase;            // [n][y_stride] running phase, then wrapped phase
  double *vuv;              // [n][y_stride] interpolated vuv (0/1)
  int *flag_cnt;            // [n][258]
  int *pulse_idx; double *pulse_shift; int *n_pulses; int pulse_cap;   // [n][pulse_cap]
  int *pulse_count;         // [n] pulses found, also those beyond pulse_cap (the host sizes the arrays from it)
  unsigned *draw_cnt; unsigned *draw_off; unsigned *draw_tot;
  const unsigned *draws;    // the context's stream table: a pulse's draws start at its draw_off entry
  double *resp;             // [n][pulse_cap][resp_n]: response i of utterance u at (u * pulse_cap + i) * resp_n
  int resp_n;               // the largest fft_size of the call
  const double *dc_remover; // [fft_size]
  double *y;
  const double2 *tw;
  int *status;
  short *y16;               // [n][y_stride] 16-bit PCM output (syn_overlap_kernel<short>), else null
  // A packed pass (null: the padded addressing above).  [n + 1] offsets from the pass's first utterance:
  const long long *f_off;   // frames: f0, sp and ap rows of utterance u start at frame f_off[u]
  const long long *s_off;   // samples: phase, vuv and y
  const long long *p_off;   // pulse slots: pulse_idx, pulse_shift, draw counts / offsets and responses (its capacity
                            // is p_off[u + 1] - p_off[u])
  const long long *cum;     // syn_pulse_kernel: [list_n + 1] first pulse of each entry of `list`; blockIdx.x is the pulse
  int list_n;               // of the launch's size group
  int n_utts;               // utterances of the pass (syn_overlap_kernel's flat grid)
};

// Where utterance u's entries start: its packed offset, or u rows of `stride` in a padded pass
WB_HD inline size_t syn_at(const long long *off, int u, size_t stride) { return off ? (size_t)off[u] : (size_t)u * stride; }

// Packed: the pass's utterances are packed (SynParams::f_off, s_off, p_off); the padded instantiation compiles without
// the offsets, as before they existed.
template <bool Packed>
WB_KERNEL(256, 2) syn_timebase_kernel(SynParams p) {
  WB_SHARED int cnt[258];
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const long long *f_off = Packed ? p.f_off : nullptr, *s_off = Packed ? p.s_off : nullptr;
  const long long *p_off = Packed ? p.p_off : nullptr;
  const int L = p.f_len[u], n = p.y_len[u], fs = p.fs;
  const double fp = p.fp_u ? p.fp_u[u] : p.frame_period;
  const int N = p.fft_u ? p.fft_u[u] : p.fft_size;
  const double lowest_f0 = fs / N + 1.0;   // synthesis.cpp:362 (integer division, then + 1.0)
  const double *f0 = p.f0 + syn_at(f_off, u, p.f_stride);
  double *phase = p.phase + syn_at(s_off, u, p.y_stride);
  double *vuv = p.vuv + syn_at(s_off, u, p.y_stride);
  const size_t p0 = syn_at(p_off, u, p.pulse_cap);
  const int cap = Packed ? (int)(p_off[u + 1] - p_off[u]) : p.pulse_cap;
  int *pidx = p.pulse_idx + p0;
  double *pshift = p.pulse_shift + p0;
  unsigned *dcnt = p.draw_cnt + p0;
  // coarse arrays are f0 thresholded; the extra point L is extrapolated (:238-245).  They are read
  // through a small accessor instead of being materialised.
#define WB_CF0(i) (f0[(i)] < lowest_f0 ? 0.0 : f0[(i)])
#define WB_CVUV(i) (WB_CF0(i) == 0.0 ? 0.0 : 1.0)
  const double f0_L = L >= 2 ? WB_CF0(L - 1) * 2 - WB_CF0(L - 2) : 0.0;
  const double vuv_L = L >= 2 ? WB_CVUV(L - 1) * 2 - WB_CVUV(L - 2) : 0.0;
  // interpolated f0 -> phase increments (kept in `phase`), interpolated vuv -> vuv
  for (int i = tid; i < n; i += nth) {
    const double t = i / static_cast<double>(fs);
    int k = (int)(t / fp);
    if (k > L) k = L;
    while (k < L + 1 && k * fp <= t) ++k;
    while (k > 0 && (k - 1) * fp > t) --k;
    k = imin(L, imax(1, k));
    const double x0 = (k - 1) * fp, x1 = k * fp;
    const double s = (t - x0) / (x1 - x0);
    const double fa = WB_CF0(k - 1), fb = (k == L) ? f0_L : WB_CF0(k);
    const double va = WB_CVUV(k - 1), vb = (k == L) ? vuv_L : WB_CVUV(k);
    const double fi = fa + s * (fb - fa), vi = va + s * (vb - va);
    const double v = vi > 0.5 ? 1.0 : 0.0;
    vuv[i] = v;
    phase[i] = 2.0 * kPi * (v == 0.0 ? 500.0 : fi) / fs;   // kDefaultF0 in unvoiced parts (:308-309)
  }
#undef WB_CF0
#undef WB_CVUV
  WB_SYNC();
  // total_phase[i] = total_phase[i-1] + increment[i], in index order (:257-262)
  if (tid == 0) {
    double run = 0.0;
    for (int i = 0; i < n; ++i) { run = (i == 0) ? phase[0] : run + phase[i]; phase[i] = run; }
  }
  WB_SYNC();
  for (int i = tid; i < n; i += nth) phase[i] = fmod(phase[i], 2.0 * kPi);
  WB_SYNC();
  // pulses: |wrap[i+1] - wrap[i]| > pi  (:265-286); ordered compaction by thread chunks
  const int chunk = (n - 1 + nth - 1) / nth;
  const int lo = imin(imax(n - 1, 0), tid * chunk), hi = imin(imax(n - 1, 0), lo + chunk);
  int c = 0;
  for (int i = lo; i < hi; ++i) c += fabs(phase[i + 1] - phase[i]) > kPi;
  cnt[tid] = c;
  WB_SYNC();
  if (tid == 0) {
    int run = 0;
    for (int t = 0; t < nth; ++t) { const int v = cnt[t]; cnt[t] = run; run += v; }
    cnt[nth] = run;
    p.n_pulses[u] = imin(run, cap);
    p.pulse_count[u] = run;   // run > cap: the host lays the chunk out again before anything reads the list
    if (run > cap) atomicOr_status(p.status, 4);   // status is null unless the counts sized this layout
  }
  WB_SYNC();
  int k = cnt[tid];
  for (int i = lo; i < hi; ++i) {
    if (fabs(phase[i + 1] - phase[i]) > kPi) {
      if (k < cap) {
        pidx[k] = i;
        const double y1 = phase[i] - 2.0 * kPi, y2 = phase[i + 1];
        pshift[k] = (-y1 / (y2 - y1)) / fs;
      }
      ++k;
    }
  }
  WB_SYNC();
  // noise_size = idx[min(np-1, i+1)] - idx[i] draws per pulse (:372-374, :19-25)
  const int np = imin(cnt[nth], cap);
  for (int i = tid; i < cap; i += nth)
    dcnt[i] = (i < np) ? (unsigned)(pidx[imin(np - 1, i + 1)] - pidx[i]) : 0u;
}

// GetMinimumPhaseSpectrum (common.cpp:192-226): log_spec[0..half] in `buf` (real, N+2 doubles),
// result (complex, half+1) left in `z` (N complex).  `buf` is destroyed.  Ends with a barrier.
WB_DEV void syn_minimum_phase(double *buf, double2 *z, int N, int lg, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH, half = N / 2;
  for (int i = half + 1 + tid; i < N; i += nth) buf[i] = buf[N - i];   // mirroring (:194-197)
  WB_SYNC();
  rfft_forward(buf, lg, tw);                                          // r2c -> cepstrum (:202)
  const double2 *c = reinterpret_cast<const double2 *>(buf);
  // cepstrum folding (:203-213), then c2c FORWARD == FFT(conj a): z[n] = conj(folded cepstrum)
  for (int i = tid; i < N; i += nth) {
    double2 v = make_double2(0.0, 0.0);
    if (i == 0 || i == half) v = make_double2(c[i].x, -c[i].y);
    else if (i < half) v = make_double2(c[i].x * 2.0, c[i].y * -2.0);
    z[i] = make_double2(v.x, -v.y);
  }
  WB_SYNC();
  cfft_forward(z, lg, tw);
  for (int i = tid; i <= half; i += nth) {                            // :220-226
    const double e = exp(z[i].x / N);
    const double a = z[i].y / N;
    z[i] = make_double2(e * cos(a), e * sin(a));
  }
  WB_SYNC();
}

// c2r (fft.cpp:26-35): out[n] = Re FFT(conj X~)[n]; X[0..half] in `spec`, work in z (N complex);
// on return z[n].x holds the unnormalised real output.  Ends with a barrier.
WB_DEV void syn_c2r(const double2 *spec, double2 *z, int N, int lg, const double2 *__restrict__ tw) {
  const int tid = WB_TID, nth = WB_NTH, half = N / 2;
  for (int i = tid; i < N; i += nth) {
    // Hermitian extension X~[N-k] = conj(X[k]); conj of it: k <= half: conj(X[k]), k > half: X[N-k]
    z[i] = (i <= half) ? make_double2(spec[i].x, -spec[i].y) : spec[N - i];
    if (i == 0 || i == half) z[i].y = 0.0;   // the reference's rdft drops Im of DC / Nyquist
  }
  WB_SYNC();
  cfft_forward(z, lg, tw);
}

template <bool Packed>
WB_KERNEL(128, 3) syn_pulse_kernel(SynParams p) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const long long *f_off = Packed ? p.f_off : nullptr, *s_off = Packed ? p.s_off : nullptr;
  const long long *p_off = Packed ? p.p_off : nullptr, *cum = Packed ? p.cum : nullptr;
  // a packed pass launches one CTA per pulse of the group: entry j of the list owns CTAs [cum[j], cum[j + 1])
  const int j = Packed ? packed_find(cum, p.list_n, (long long)blockIdx.x) : (int)blockIdx.y;
  const int u = p.list ? p.list[j] : j, pi = Packed ? (int)(blockIdx.x - cum[j]) : (int)blockIdx.x;
  const int np = p.n_pulses[u];
  if (pi >= np) return;
  const int N = p.fft_size, half = N / 2, lg = p.lg_fft, fs = p.fs;
  double2 *z = reinterpret_cast<double2 *>(smem);                 // N complex
  double2 *mps = z + N;                                           // half + 1 complex (+pad)
  double *buf = reinterpret_cast<double *>(mps + (half + 2));     // N + 2 doubles
  double *env = buf + (N + 2);                                    // half + 1
  double *apr = env + (half + 1);                                 // half + 1
  double *per = apr + (half + 1);                                 // N: periodic response
  double *red = per + N;                                          // WB_RED_DOUBLES

  const int L = p.f_len[u];
  const size_t p0 = syn_at(p_off, u, p.pulse_cap);
  const int idx = p.pulse_idx[p0 + pi];
  const int idx_next = p.pulse_idx[p0 + imin(np - 1, pi + 1)];
  const int noise_size = idx_next - idx;
  const double shift = p.pulse_shift[p0 + pi];
  const double current_vuv = p.vuv[syn_at(s_off, u, p.y_stride) + idx];
  const double current_time = idx / static_cast<double>(fs);
  double *resp = p.resp + (p0 + pi) * p.resp_n;
  const size_t bins = p.row;
  const size_t r0 = syn_at(f_off, u, p.f_stride) * bins;
  const double *sp = p.sp + r0, *ap = p.ap + r0;

  // GetSpectralEnvelope / GetAperiodicRatio (:140-179)
  const double fp = p.fp_u ? p.fp_u[u] : p.frame_period;
  const int fl = imin(L - 1, static_cast<int>(floor(current_time / fp)));
  const int ce = imin(L - 1, static_cast<int>(ceil(current_time / fp)));
  const double interp = current_time / fp - fl;
  for (int k = tid; k <= half; k += nth) {
    double e, a;
    const double a0 = dmax(0.001, dmin(0.999999999999, ap[fl * bins + k]));
    if (fl == ce) {
      e = fabs(sp[fl * bins + k]);
      a = pow(a0, 2.0);
    } else {
      const double a1 = dmax(0.001, dmin(0.999999999999, ap[ce * bins + k]));
      e = (1.0 - interp) * fabs(sp[fl * bins + k]) + interp * fabs(sp[ce * bins + k]);
      a = pow((1.0 - interp) * a0 + interp * a1, 2.0);
    }
    env[k] = e; apr[k] = a;
  }
  WB_SYNC();

  // ---- periodic response (:110-138)
  const bool voiced_pulse = !(current_vuv <= 0.5 || apr[0] > 0.999);
  if (voiced_pulse) {
    for (int k = tid; k <= half; k += nth) buf[k] = log(env[k] * (1.0 - apr[k]) + kTiny) / 2.0;
    WB_SYNC();
    syn_minimum_phase(buf, z, N, lg, p.tw);
    const double coefficient = 2.0 * kPi * shift * fs / N;
    for (int k = tid; k <= half; k += nth) {                     // fractional time shift (:93-105)
      const double re = z[k].x, im = z[k].y;
      const double re2 = cos(coefficient * k);
      const double im2 = sqrt(1.0 - re2 * re2);
      mps[k] = make_double2(re * re2 + im * im2, im * re2 - re * im2);
    }
    WB_SYNC();
    syn_c2r(mps, z, N, lg, p.tw);
    // fftshift (matlabfunctions.cpp:73-78) then RemoveDCComponent (:75-85)
    double dc = 0.0;
    for (int i = tid; i < half; i += nth) dc += z[i].x;          // shifted[half + i] = waveform[i]
    dc = block_sum(dc, red);
    for (int i = tid; i < N; i += nth) {
      const double shifted = (i < half) ? z[i + half].x : z[i - half].x;
      per[i] = (i < half) ? -dc * __ldg(&p.dc_remover[i]) : shifted - dc * __ldg(&p.dc_remover[i]);
    }
  } else {
    for (int i = tid; i < N; i += nth) per[i] = 0.0;
  }
  WB_SYNC();

  // ---- aperiodic response (:36-69).  The last pulse (noise_size 0) runs it too: its noise is all zeros and sqrt(0)
  // scales the periodic part away, which gives zeros where both responses are finite and NaN where either is not (a
  // zero envelope's log(0)), as in the reference.
  const unsigned *draw = p.draws + p.draw_off[p0 + pi];
  double s = 0.0;
  for (int i = tid; i < N + 2; i += nth) {
    const double v = (i < noise_size && i < N) ? randn_value(draw[i]) : 0.0;
    buf[i] = v;
    s += v;
  }
  const double average = block_sum(s, red) / noise_size;
  for (int i = tid; i < noise_size && i < N; i += nth) buf[i] -= average;
  WB_SYNC();
  rfft_forward(buf, lg, p.tw);
  const double2 *ns = reinterpret_cast<const double2 *>(buf);
  for (int k = tid; k <= half; k += nth) mps[k] = ns[k];        // keep the noise spectrum
  WB_SYNC();
  for (int k = tid; k <= half; k += nth)
    buf[k] = (current_vuv != 0.0) ? log(env[k] * apr[k]) / 2.0 : log(env[k]) / 2.0;
  WB_SYNC();
  syn_minimum_phase(buf, z, N, lg, p.tw);
  for (int k = tid; k <= half; k += nth) {
    const double2 m = z[k], q = mps[k];
    mps[k] = make_double2(m.x * q.x - m.y * q.y, m.x * q.y + m.y * q.x);
  }
  WB_SYNC();
  syn_c2r(mps, z, N, lg, p.tw);
  const double sq = sqrt(static_cast<double>(noise_size));
  for (int i = tid; i < N; i += nth) {
    const double aper = (i < half) ? z[i + half].x : z[i - half].x;   // fftshift
    resp[i] = (per[i] * sq + aper) / N;                                // :214-217
  }
}

// wavwrite's quantisation (tools/audioio.cpp:163-165, wb_fileio.cu wavwrite): (int)(v * 32767) truncated toward zero,
// then clamped to [-32768, 32767].  Where the product does not fit an int the reference's cast is undefined; here it
// saturates by sign, and NaN gives 0.
WB_HD inline short pcm16_of(double v) {
  const double s = v * 32767;
  if (!(s == s)) return 0;
  if (s >= 32767.0) return 32767;
  if (s <= -32768.0) return -32768;
  return static_cast<short>(static_cast<int>(s));
}

// Out = double: the waveform (p.y); Out = short: its 16-bit PCM (p.y16), the sum never reaching memory
// Padded: (sample, utterance) -> thread over a (max_y, n) grid.  Packed: one flat grid over the pass's samples, each
// thread finding its utterance in s_off.
template <typename Out>
WB_KERNEL_PLAIN syn_overlap_kernel(SynParams p) {
  int u, s;
  if (p.s_off) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= p.s_off[p.n_utts]) return;
    u = packed_find(p.s_off, p.n_utts, g);
    s = (int)(g - p.s_off[u]);
  } else {
    u = blockIdx.y;
    s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= p.y_len[u]) return;
  }
  const int N = p.fft_u ? p.fft_u[u] : p.fft_size, half = N / 2, np = p.n_pulses[u];
  const size_t p0 = syn_at(p.p_off, u, p.pulse_cap);
  const int *pidx = p.pulse_idx + p0;
  // pulse i covers samples idx_i - half + 1 .. idx_i + half  ->  idx_i in [s - half, s + half - 1]
  int lo = 0, hi = np;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (pidx[mid] < s - half) lo = mid + 1; else hi = mid; }
  double acc = 0.0;
  for (int i = lo; i < np && pidx[i] <= s + half - 1; ++i) {
    const int j = s - (pidx[i] - half + 1);
    acc += p.resp[(p0 + i) * p.resp_n + j];
  }
  const size_t at = syn_at(p.s_off, u, p.y_stride) + s;
  if constexpr (std::is_same<Out, short>::value) p.y16[at] = pcm16_of(acc);
  else p.y[at] = acc;
}

// ---- voice modification --------------------------------------------------------------------------------------------
// F0 scaling and formant shift over a batch: the reference demo's ParameterModification (test/test.cpp:221-258), the
// step a vocoder sits between analysis and synthesis for.  world_b200_modify_batch runs it on full rows; synthesis_run
// runs the same two kernels on each pass's f0 copy and decoded envelope block.
//
// Per utterance, with shift (f0 factor) and ratio (spectral stretch), half = fft_size / 2, bins = half + 1:
//   f0[i] *= shift
//   x[i] = ratio * i / fft_size * fs,  xi[j] = (double)j / fft_size * fs,  L[m] = log(sp[m])
//   sp[j] = exp(interp1(x, L, xi)[j])        (histc, then y[k-1] + s * (y[k] - y[k-1]), extrapolating)
//   ratio < 1: sp[j] = sp[c - 1] for j >= c = (int)(fft_size / 2.0 * ratio)
// The segment k and the weight s of every bin depend on (ratio, fft_size, fs) only.  They are planned on the host
// with the reference's expressions and the library's own histc (wb_matlab.cu), one table per distinct (ratio,
// fft_size), and the tail rule is folded in (entry j := entry c - 1 gives the same value).  The kernel is then one
// gather per bin:
//   modify_stretch_kernel  (frame, utterance) -> CTA: the row's logs into shared memory, barrier,
//                          out[j] = exp(L[a] + s * (L[a + 1] - L[a])), rounded step by step as the reference's
//                          unfused x86-64 build rounds it
//   modify_f0_kernel       frame -> thread: f0 * shift

#define WB_MODIFY_THREADS 128

// Rows of frames >= f_len[u] (and utterances >= n_utts) are never touched.  The `continue` is uniform over the CTA.
// Each frame row holds `row` doubles, of which the utterance's table covers the first tbins[t].
// f_off: [n_utts + 1] frame offsets of packed rows (utterance u's frame f at row f_off[u] + f), or null: padded rows.
WB_KERNEL(WB_MODIFY_THREADS, 8) modify_stretch_kernel(double *sp, const int *__restrict__ f_len, int n_utts,
                                                      int f_stride, int row_len, const int *__restrict__ table,
                                                      const int *__restrict__ tbins, const int *__restrict__ toff,
                                                      const int *__restrict__ idx, const double *__restrict__ frac,
                                                      const long long *__restrict__ f_off) {
  WB_DYN_SMEM(double, logs);   // the largest table's bins
  const int tid = WB_TID, nth = WB_NTH, f = blockIdx.x;
  for (int u = blockIdx.y; u < n_utts; u += gridDim.y) {
    if (f >= f_len[u]) continue;
    double *row = sp + (syn_at(f_off, u, f_stride) + f) * row_len;
    const int t = __ldg(&table[u]), bins = __ldg(&tbins[t]);
    const size_t t0 = (size_t)__ldg(&toff[t]);
    for (int j = tid; j < bins; j += nth) logs[j] = log(row[j]);
    WB_SYNC();
    for (int j = tid; j < bins; j += nth) {
      const int a = __ldg(&idx[t0 + j]);
      const double s = __ldg(&frac[t0 + j]);
      const double la = logs[a], lb = logs[a + 1];
      // y[k-1] + s * (y[k] - y[k-1]) (matlabfunctions.cpp:171): three roundings, no FMA
      row[j] = exp(__dadd_rn(la, __dmul_rn(s, __dsub_rn(lb, la))));
    }
    WB_SYNC();
  }
}

WB_KERNEL_PLAIN modify_f0_kernel(const double *f0_in, double *f0_out, const double *__restrict__ scale,
                                 const int *__restrict__ f_len, int n_utts, int f_stride,
                                 const long long *__restrict__ f_off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int u = blockIdx.y; u < n_utts; u += gridDim.y)
    if (i < f_len[u]) {
      const size_t at = syn_at(f_off, u, f_stride) + i;
      f0_out[at] = __dmul_rn(f0_in[at], scale[u]);
    }
}

// ---- pitch and formant curves: one f0 factor and one spectral ratio per frame ----------------------------------------
// Frame i of an utterance is modified as ParameterModification modifies a one-frame spectrogram with shift =
// f0_curve[i] and ratio = ratio_curve[i] at the utterance's fft_size.  A (ratio, fft_size) table per frame would be
// 12 bytes per bin per frame, so the stretch works out each frame's segments and weights on the device instead, with
// modify_plan's expressions in modify_plan's order (every step rounded on its own: no FMA):
//   modify_curve_stretch_kernel  frame -> CTA.  Padded rows: the (frame, utterance) grid of modify_stretch_kernel;
//                                packed rows: one CTA per packed frame, the utterance found by packed_find.  The CTA
//                                builds x[i] = ratio * i / n_fft * fs and L[i] = log(sp[i]) in shared memory, then per
//                                bin j (j := c - 1 past the tail c = (int)(n_fft / 2.0 * ratio) when ratio < 1, as
//                                modify_plan folds it) takes xi = (double)j / n_fft * fs, its histc segment k, s =
//                                (xi - x[k - 1]) / (x[k] - x[k - 1]) and exp(L[a] + s * (L[a + 1] - L[a])) with the
//                                three roundings of modify_stretch_kernel.  On constant curves each row equals
//                                modify_stretch_kernel's bit for bit.
//   modify_curve_f0_kernel       frame -> thread: f0 * curve, rounded as modify_f0_kernel
//   modify_curve_check_kernel    frame -> thread: the first frame of each curve that breaks modify_plan's rule
//                                (atomicMin on its index), read back once by the host before any modification.
// Segment search: histc (wb_matlab.cu) walks the edges and nodes in step.  For a strictly ascending x (ratio > 0:
// consecutive nodes differ by ratio * fs / n_fft, far above an ulp) and ascending edges xi, the bin it gives edge xi is
//   k = min(bins - 1, the first b >= 1 with xi < x[b])
// (an edge below x[1] stays in bin 1; the walk advances past node b exactly when xi >= x[b]; past the last node every
// edge is bin bins - 1).  That is a binary search over x in shared memory, about log2(bins) loads per bin.  Where xi
// equals a node (ratios 0.5, 1.0, 2.0 put edges on nodes), xi < x[b] is false at that node, so the edge goes to the
// segment that starts there, as in histc.

WB_DEV void curve_stretch_row(double *row, int n_fft, int fs, double ratio, double *x, double *logs) {
  const int tid = WB_TID, nth = WB_NTH, bins = n_fft / 2 + 1;
  const double nf = (double)n_fft, fsd = (double)fs;
  for (int i = tid; i < bins; i += nth) {   // test.cpp:237-240 as modify_plan: ((ratio * i) / n_fft) * fs
    x[i] = __dmul_rn(__ddiv_rn(__dmul_rn(ratio, (double)i), nf), fsd);
    logs[i] = log(row[i]);
  }
  WB_SYNC();
  const int c = ratio < 1.0 ? static_cast<int>(n_fft / 2.0 * ratio) : bins;   // test.cpp:250-254
  for (int j = tid; j < bins; j += nth) {
    const int e = j < c ? j : c - 1;
    const double xi = __dmul_rn(__ddiv_rn((double)e, nf), fsd);
    int lo = 1, hi = bins - 1;   // the first b in [1, bins - 1] with xi < x[b], else bins - 1
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (xi < x[mid]) hi = mid; else lo = mid + 1;
    }
    const int a = lo - 1;
    const double s = __dsub_rn(xi, x[a]) / __dsub_rn(x[a + 1], x[a]);   // matlabfunctions.cpp:162-171
    const double la = logs[a], lb = logs[a + 1];
    row[j] = exp(__dadd_rn(la, __dmul_rn(s, __dsub_rn(lb, la))));
  }
  WB_SYNC();
}

// fft_u: [n_utts] each utterance's fft_size; ratio: the curve, indexed like the frames' rows.  f_off null: padded rows,
// grid (max_f, utterances); else packed rows, frames [0, frames) over a 1-D grid.  Dynamic shared memory: 2 * max_bins
// doubles.
WB_KERNEL(WB_MODIFY_THREADS, 8) modify_curve_stretch_kernel(double *sp, const int *__restrict__ f_len, int n_utts,
                                                            int f_stride, int row_len, const int *__restrict__ fft_u,
                                                            int fs, const double *__restrict__ ratio,
                                                            const long long *__restrict__ f_off, long long frames,
                                                            int max_bins) {
  WB_DYN_SMEM(double, x);
  double *logs = x + max_bins;
  if (f_off) {
    for (long long g = blockIdx.x; g < frames; g += gridDim.x) {
      const int u = packed_find(f_off, n_utts, g);
      curve_stretch_row(sp + (size_t)g * row_len, __ldg(&fft_u[u]), fs, __ldg(&ratio[g]), x, logs);
    }
    return;
  }
  const int f = blockIdx.x;
  for (int u = blockIdx.y; u < n_utts; u += gridDim.y) {
    if (f >= f_len[u]) continue;   // uniform over the CTA
    const size_t at = (size_t)u * f_stride + f;
    curve_stretch_row(sp + at * row_len, __ldg(&fft_u[u]), fs, __ldg(&ratio[at]), x, logs);
  }
}

WB_KERNEL_PLAIN modify_curve_f0_kernel(double *f0, const double *__restrict__ curve, const int *__restrict__ f_len,
                                       int n_utts, int f_stride, const long long *__restrict__ f_off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int u = blockIdx.y; u < n_utts; u += gridDim.y)
    if (i < f_len[u]) {
      const size_t at = syn_at(f_off, u, f_stride) + i;
      f0[at] = __dmul_rn(f0[at], curve[at]);
    }
}

// modify_plan's rules for one value (f0: a finite factor > 0; ratio: also c = (int)(n_fft / 2.0 * r) >= 1 below 1)
WB_HD inline bool curve_f0_bad(double v) { return !(v > 0.0) || !isfinite(v); }
WB_HD inline bool curve_ratio_bad(double r, int n_fft) {
  return !(r > 0.0) || !isfinite(r) || (r < 1.0 && static_cast<int>(n_fft / 2.0 * r) < 1);
}

// first[0] / first[1]: the smallest index of a bad f0 / ratio value (ULLONG_MAX on entry: none)
WB_KERNEL_PLAIN modify_curve_check_kernel(const double *__restrict__ f0c, const double *__restrict__ ratio,
                                          const int *__restrict__ f_len, int n_utts, int f_stride,
                                          const int *__restrict__ fft_u, const long long *__restrict__ f_off,
                                          unsigned long long *first) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int u = blockIdx.y; u < n_utts; u += gridDim.y)
    if (i < f_len[u]) {
      const size_t at = syn_at(f_off, u, f_stride) + i;
      if (f0c && curve_f0_bad(f0c[at])) atomicMin(&first[0], (unsigned long long)at);
      if (ratio && curve_ratio_bad(ratio[at], fft_u[u])) atomicMin(&first[1], (unsigned long long)at);
    }
}

namespace {
struct ModifyLayout {
  size_t o_idx, o_frac, o_tbins, o_toff, o_scale, o_table, total;
  ModifyLayout(const ModifyPlan &p, int n) {
    ArenaPlan a;
    const size_t cells = p.idx.size();
    o_idx = a.add(cells * 4); o_frac = a.add(cells * 8);
    o_tbins = a.add((size_t)p.n_tables * 4); o_toff = a.add((size_t)p.n_tables * 4);
    o_scale = a.add(p.scale.empty() ? 0 : (size_t)n * 8); o_table = a.add(p.table.empty() ? 0 : (size_t)n * 4);
    total = a.total;
  }
};

int modify_fail(Ctx *ctx, const char *who, const char *what, int u, double v, const char *why) {
  char msg[256];
  snprintf(msg, sizeof msg, "%s: %s[%d] = %.17g %s", who, what, u, v, why);
  ctx->last_error = msg;
  return WORLD_B200_EINVAL;
}
}  // namespace

size_t ModifyPlan::device_bytes(int n) const { return ModifyLayout(*this, n).total; }

int modify_plan(Ctx *ctx, const char *who, int n_utts, int fft_size, int fs, const double *f0_scale,
                const double *spectral_ratio, ModifyPlan *plan, const int *fft_sizes) {
  *plan = ModifyPlan();
  if (f0_scale) {
    for (int u = 0; u < n_utts; ++u) {
      const double v = f0_scale[u];
      if (!(v > 0.0) || !isfinite(v)) return modify_fail(ctx, who, "f0_scale", u, v, "is not a finite factor > 0");
    }
    plan->scale.assign(f0_scale, f0_scale + n_utts);
  }
  if (!spectral_ratio) return 0;
  if (!fft_sizes && (fft_size < 16 || fft_size > 4096 || (fft_size & (fft_size - 1)))) {
    ctx->last_error = std::string(who) + ": fft_size must be a power of two in [16, 4096]";
    return WORLD_B200_EINVAL;
  }
  if (fs <= 0) {
    ctx->last_error = std::string(who) + ": fs must be > 0";
    return WORLD_B200_EINVAL;
  }
  for (int u = 0; u < n_utts; ++u) {
    const double r = spectral_ratio[u];
    const int n_fft = fft_sizes ? fft_sizes[u] : fft_size;
    // histc needs an ascending axis; below 1 the tail copies bin c - 1, which must exist (c == 0 reads sp[-1])
    if (!(r > 0.0) || !isfinite(r)) return modify_fail(ctx, who, "spectral_ratio", u, r, "is not a finite ratio > 0");
    if (r < 1.0 && static_cast<int>(n_fft / 2.0 * r) < 1)
      return modify_fail(ctx, who, "spectral_ratio", u, r, "leaves no bin below (int)(fft_size / 2.0 * ratio)");
  }
  plan->table.resize(n_utts);
  std::map<std::pair<double, int>, int> seen;
  std::vector<double> x, xi;
  std::vector<int> k;
  for (int u = 0; u < n_utts; ++u) {
    const double ratio = spectral_ratio[u];
    const int n_fft = fft_sizes ? fft_sizes[u] : fft_size, half = n_fft / 2, bins = half + 1;
    auto it = seen.find({ratio, n_fft});
    if (it != seen.end()) { plan->table[u] = it->second; continue; }
    const int t = plan->n_tables++;
    seen[{ratio, n_fft}] = t;
    plan->table[u] = t;
    plan->bins = imax(plan->bins, bins);
    plan->tbins.push_back(bins);
    plan->toff.push_back((int)plan->idx.size());
    x.resize(bins); xi.resize(bins); k.resize(bins);
    for (int i = 0; i <= half; ++i) {   // test.cpp:237-240, the same expressions in the same order
      x[i] = ratio * i / n_fft * fs;
      xi[i] = static_cast<double>(i) / n_fft * fs;
    }
    histc(x.data(), bins, xi.data(), bins, k.data());
    plan->idx.resize(plan->idx.size() + bins);
    plan->frac.resize(plan->frac.size() + bins);
    int *ia = plan->idx.data() + plan->toff[t];
    double *sa = plan->frac.data() + plan->toff[t];
    for (int j = 0; j < bins; ++j) {   // matlabfunctions.cpp:162-171: h[k-1] = x[k] - x[k-1], s = (xi - x[k-1]) / h
      const int a = k[j] - 1;
      ia[j] = a;
      sa[j] = (xi[j] - x[a]) / (x[a + 1] - x[a]);
    }
    if (ratio < 1.0) {                 // test.cpp:250-254
      const int c = static_cast<int>(n_fft / 2.0 * ratio);
      for (int j = c; j < bins; ++j) { ia[j] = ia[c - 1]; sa[j] = sa[c - 1]; }
    }
  }
  return 0;
}

int modify_upload(Ctx *ctx, const ModifyPlan &plan, int u0, int n, unsigned char *blk, ModifyDevice *d) {
  const ModifyLayout l(plan, n);
  int rc = 0;
  if (!plan.idx.empty()) rc = dev_memcpy_h2d(ctx, blk + l.o_idx, plan.idx.data(), plan.idx.size() * 4);
  if (!rc && !plan.frac.empty()) rc = dev_memcpy_h2d(ctx, blk + l.o_frac, plan.frac.data(), plan.frac.size() * 8);
  if (!rc && plan.n_tables) rc = dev_memcpy_h2d(ctx, blk + l.o_tbins, plan.tbins.data(), (size_t)plan.n_tables * 4);
  if (!rc && plan.n_tables) rc = dev_memcpy_h2d(ctx, blk + l.o_toff, plan.toff.data(), (size_t)plan.n_tables * 4);
  if (!rc && !plan.scale.empty()) rc = dev_memcpy_h2d(ctx, blk + l.o_scale, plan.scale.data() + u0, (size_t)n * 8);
  if (!rc && !plan.table.empty()) rc = dev_memcpy_h2d(ctx, blk + l.o_table, plan.table.data() + u0, (size_t)n * 4);
  d->idx = (const int *)(blk + l.o_idx); d->frac = (const double *)(blk + l.o_frac);
  d->scale = (const double *)(blk + l.o_scale); d->table = (const int *)(blk + l.o_table);
  d->tbins = (const int *)(blk + l.o_tbins); d->toff = (const int *)(blk + l.o_toff);
  return rc;
}

void modify_f0_launch(Ctx *ctx, const ModifyDevice &d, const int *f_len, int n_utts, int f_stride, int max_f,
                      const double *f0_in, double *f0_out, const long long *f_off) {
  if (n_utts <= 0 || max_f <= 0) return;
  const dim3 grid((unsigned)((max_f + 255) / 256), (unsigned)imin(n_utts, 65535));
  WB_LAUNCH_FLAT(modify_f0_kernel, grid, 256, 0, ctx->stream, f0_in, f0_out, d.scale, f_len, n_utts, f_stride, f_off);
}

void modify_stretch_launch(Ctx *ctx, const ModifyDevice &d, int row, int max_bins, const int *f_len, int n_utts,
                           int f_stride, int max_f, double *spectrogram, const long long *f_off) {
  if (n_utts <= 0 || max_f <= 0) return;
  const dim3 grid((unsigned)max_f, (unsigned)imin(n_utts, 65535));
  WB_LAUNCH_COOP(modify_stretch_kernel, grid, WB_MODIFY_THREADS, (size_t)max_bins * 8, ctx->stream, spectrogram, f_len,
                 n_utts, f_stride, row, d.table, d.tbins, d.toff, d.idx, d.frac, f_off);
}

int modify_run(Ctx *ctx, const ModifyPlan &plan, int u0, int n_utts, const int *f0_lengths, int f0_stride, int row,
               double *f0, double *spectrogram, const long long *f_offsets) {
  int max_f = 0;
  for (int u = 0; u < n_utts; ++u) max_f = imax(max_f, f0_lengths[u]);
  if (max_f == 0 || (plan.scale.empty() && plan.table.empty())) return 0;
  ArenaPlan a;
  const size_t o_len = a.add((size_t)n_utts * 4), o_mod = a.add(plan.device_bytes(n_utts));
  const size_t o_off = a.add(f_offsets ? (size_t)(n_utts + 1) * 8 : 0);
  unsigned char *blk = arena_block(ctx, a.total);
  if (!blk) return WORLD_B200_ENOMEM;
  ModifyDevice d;
  int rc = dev_memcpy_h2d(ctx, blk + o_len, f0_lengths, (size_t)n_utts * 4);
  if (!rc) rc = modify_upload(ctx, plan, u0, n_utts, blk + o_mod, &d);
  if (!rc && f_offsets) rc = dev_memcpy_h2d(ctx, blk + o_off, f_offsets, (size_t)(n_utts + 1) * 8);
  if (rc) return rc;
  const int *f_len = (const int *)(blk + o_len);
  const long long *f_off = f_offsets ? (const long long *)(blk + o_off) : nullptr;
  if (!plan.scale.empty()) modify_f0_launch(ctx, d, f_len, n_utts, f0_stride, max_f, f0, f0, f_off);
  if (!plan.table.empty())
    modify_stretch_launch(ctx, d, row, plan.bins, f_len, n_utts, f0_stride, max_f, spectrogram, f_off);
  return dev_check(ctx, "modify");
}

namespace {
// The rows' lengths, sizes and (packed) offsets on the device, in one arena block with `extra` bytes after them
struct CurveRows {
  const int *f_len, *fft; const long long *f_off; unsigned char *extra;
  int max_f; long long frames;
};
int curve_rows(Ctx *ctx, int n_utts, const int *f_len, int f_stride, const long long *f_off, const int *fft_sizes,
               size_t extra, CurveRows *d) {
  d->max_f = 0;
  for (int u = 0; u < n_utts; ++u) d->max_f = imax(d->max_f, f_len[u]);
  d->frames = f_off ? f_off[n_utts] : (long long)n_utts * f_stride;
  ArenaPlan a;
  const size_t o_len = a.add((size_t)n_utts * 4), o_fft = a.add(fft_sizes ? (size_t)n_utts * 4 : 0);
  const size_t o_off = a.add(f_off ? (size_t)(n_utts + 1) * 8 : 0), o_extra = a.add(extra);
  unsigned char *blk = arena_block(ctx, a.total);
  if (!blk) return WORLD_B200_ENOMEM;
  int rc = dev_memcpy_h2d(ctx, blk + o_len, f_len, (size_t)n_utts * 4);
  if (!rc && fft_sizes) rc = dev_memcpy_h2d(ctx, blk + o_fft, fft_sizes, (size_t)n_utts * 4);
  if (!rc && f_off) rc = dev_memcpy_h2d(ctx, blk + o_off, f_off, (size_t)(n_utts + 1) * 8);
  d->f_len = (const int *)(blk + o_len);
  d->fft = fft_sizes ? (const int *)(blk + o_fft) : nullptr;
  d->f_off = f_off ? (const long long *)(blk + o_off) : nullptr;
  d->extra = blk + o_extra;
  return rc;
}

// EINVAL naming the curve value at index `at` of the rows: its utterance and frame
int curve_fail(Ctx *ctx, const char *who, bool ratio, long long at, int n_utts, int f_stride, const long long *f_off,
               double v) {
  const int u = f_off ? packed_find(f_off, n_utts, at) : (int)(at / f_stride);
  const long long f = f_off ? at - f_off[u] : at % f_stride;
  char msg[320];
  snprintf(msg, sizeof msg, "%s: %s[%lld] = %.17g (utterance %d, frame %lld) %s", who,
           ratio ? "spectral_ratio_curve" : "f0_curve", at, v, u, f,
           ratio ? "is not a finite ratio > 0 that leaves a bin below (int)(fft_size / 2.0 * ratio)"
                 : "is not a finite factor > 0");
  ctx->last_error = msg;
  return WORLD_B200_EINVAL;
}
}  // namespace

int curves_check(Ctx *ctx, const char *who, const ModifyCurves &cv, int n_utts, const int *f_len, int f_stride,
                 const long long *f_off, const int *fft_sizes) {
  if (n_utts <= 0 || (!cv.f0 && !cv.ratio)) return 0;
  CurveRows d;
  int rc = curve_rows(ctx, n_utts, f_len, f_stride, f_off, cv.ratio ? fft_sizes : nullptr, 16, &d);
  if (rc || d.max_f == 0) return rc;
  unsigned long long *first = (unsigned long long *)d.extra, got[2];
  rc = dev_memset(ctx, first, 0xff, 16);
  if (rc) return rc;
  const dim3 grid((unsigned)((d.max_f + 255) / 256), (unsigned)imin(n_utts, 65535));
  WB_LAUNCH_FLAT(modify_curve_check_kernel, grid, 256, 0, ctx->stream, cv.f0, cv.ratio, d.f_len, n_utts, f_stride,
                 d.fft, d.f_off, first);
  rc = dev_check(ctx, "modify curves check");
  if (!rc) rc = dev_memcpy_d2h(ctx, got, first, 16);
  if (!rc) rc = dev_sync(ctx);
  for (int k = 0; k < 2 && !rc; ++k) {
    if (got[k] == ~0ull) continue;
    double v = 0.0;
    rc = dev_memcpy_d2h(ctx, &v, (k ? cv.ratio : cv.f0) + got[k], 8);
    if (!rc) rc = dev_sync(ctx);
    if (!rc) rc = curve_fail(ctx, who, k == 1, (long long)got[k], n_utts, f_stride, f_off, v);
  }
  return rc;
}

int curves_check_host(Ctx *ctx, const char *who, const ModifyCurves &cv, int n_utts, const int *f_len, int f_stride,
                      const long long *f_off, const int *fft_sizes) {
  for (int k = 0; k < 2; ++k) {
    const double *c = k ? cv.ratio : cv.f0;
    for (int u = 0; u < n_utts && c; ++u)
      for (int i = 0; i < f_len[u]; ++i) {
        const long long at = (long long)syn_at(f_off, u, f_stride) + i;
        if (k ? curve_ratio_bad(c[at], fft_sizes[u]) : curve_f0_bad(c[at]))
          return curve_fail(ctx, who, k == 1, at, n_utts, f_stride, f_off, c[at]);
      }
  }
  return 0;
}

int curves_run(Ctx *ctx, const ModifyCurves &cv, int n_utts, const int *f_len, int f_stride, const long long *f_off,
               const int *fft_sizes, int fs, int row, double *f0, double *spectrogram) {
  const bool scale = cv.f0 && f0, stretch = cv.ratio && spectrogram;
  if (n_utts <= 0 || (!scale && !stretch)) return 0;
  CurveRows d;
  int rc = curve_rows(ctx, n_utts, f_len, f_stride, f_off, stretch ? fft_sizes : nullptr, 0, &d);
  if (rc || d.max_f == 0) return rc;
  if (scale) {
    const dim3 grid((unsigned)((d.max_f + 255) / 256), (unsigned)imin(n_utts, 65535));
    WB_LAUNCH_FLAT(modify_curve_f0_kernel, grid, 256, 0, ctx->stream, f0, cv.f0, d.f_len, n_utts, f_stride, d.f_off);
  }
  if (stretch) {
    int max_bins = 0;
    for (int u = 0; u < n_utts; ++u) max_bins = imax(max_bins, fft_sizes[u] / 2 + 1);
    const dim3 grid = f_off ? dim3((unsigned)std::min<long long>(d.frames, INT_MAX))
                            : dim3((unsigned)d.max_f, (unsigned)imin(n_utts, 65535));
    if (d.frames > 0)
      WB_LAUNCH_COOP(modify_curve_stretch_kernel, grid, WB_MODIFY_THREADS, (size_t)max_bins * 16, ctx->stream,
                     spectrogram, d.f_len, n_utts, f_stride, row, d.fft, fs, cv.ratio, d.f_off, d.frames, max_bins);
  }
  return dev_check(ctx, "modify curves");
}

int row_lengths(Ctx *ctx, const char *who, const char *rows, const int *lengths, int n, int stride, int least,
                std::vector<int> *out) {
  out->resize(n);
  for (int u = 0; u < n; ++u) {
    const int v = (*out)[u] = lengths ? lengths[u] : stride;
    if (v < least || v > stride) {
      char msg[256];
      snprintf(msg, sizeof msg, "%s: %s_lengths[%d] = %d is outside [%d, %s_stride = %d] (utterance %d)", who, rows,
               u, v, least, rows, stride, u);
      ctx->last_error = msg;
      return WORLD_B200_EINVAL;
    }
  }
  return 0;
}

// Packed rows: utterance u is entries [off[u], off[u + 1]) of the `rows` arrays; out[u] = its count.  The rule of
// packed_lengths (wb_api.cu); EINVAL with last_error "<who>: " and its message for the first utterance that breaks it.
int packed_lengths(Ctx *ctx, const char *who, const char *rows, const char *what, const long long *off, int n,
                   int least, std::vector<int> *out) {
  const std::string bad = packed_lengths((std::string(rows) + "_offsets").c_str(), what, n, off, least, out);
  if (bad.empty()) return 0;
  ctx->last_error = std::string(who) + ": " + bad;
  return WORLD_B200_EINVAL;
}

int synthesis_plan(Ctx *ctx, const SynthesisRequest &r, const char *who, SynthesisPlan *p) {
  auto fail = [&](const std::string &what) {
    ctx->last_error = std::string(who) + ": " + what;
    return WORLD_B200_EINVAL;
  };
  auto fail_u = [&](const std::string &what, int u) { return fail(what + " (utterance " + std::to_string(u) + ")"); };
  if (!r.y || (!r.transform && (!r.f0 || !r.sp || (!r.coded && !r.ap))))
    return fail(r.coded ? "f0, coded_spectral_envelope and y must be given"
                        : "f0, spectrogram, aperiodicity and y must be given");
  if (r.per_utt && !r.fft_sizes) return fail("fft_sizes must be given");
  const bool packed = r.f_offsets || r.y_offsets;
  if (packed && (!r.f_offsets || !r.y_offsets)) return fail("f_offsets and y_offsets must be given");
  if (r.n < 0) return fail("n_utts must be >= 0");
  if (r.fs <= 0) return fail("fs must be > 0");
  if (r.frame_period <= 0) return fail("frame_period must be > 0");
  if (r.nbit != 0 && r.nbit != 16) return fail("nbit must be 0 (double) or 16 (int16)");
  auto bad_size = [](int f) { return f < 16 || f > WB_TW_N / 2 || (f & (f - 1)); };
  if (!r.per_utt && bad_size(r.fft_size)) return fail("fft_size must be a power of two in [16, 4096]");
  // each utterance's size, and the distinct sizes in order of first appearance
  p->size.assign(r.n, 0);
  if (!r.per_utt) p->sizes.assign(1, r.fft_size);
  for (int u = 0; u < r.n && r.per_utt; ++u) {
    const int f = r.fft_sizes[u];
    if (bad_size(f))
      return fail_u("fft_sizes[" + std::to_string(u) + "] = " + std::to_string(f) +
                    " is not a power of two in [16, 4096]", u);
    const auto it = std::find(p->sizes.begin(), p->sizes.end(), f);
    p->size[u] = (int)(it - p->sizes.begin());
    if (it == p->sizes.end()) p->sizes.push_back(f);
  }
  p->fft_size = 0;
  for (const int f : p->sizes) p->fft_size = imax(p->fft_size, f);
  p->row = p->fft_size / 2 + 1;
  if (r.per_utt && !r.coded) {
    // packed rows of row_stride 0: the largest size's bins, as the packed analysis writes them
    const int row_stride = packed && r.row_stride == 0 ? p->row : r.row_stride;
    p->row = row_stride;
    for (int u = 0; u < r.n; ++u)
      if (row_stride < r.fft_sizes[u] / 2 + 1)
        return fail_u("row_stride = " + std::to_string(row_stride) + " is smaller than fft_sizes[" +
                      std::to_string(u) + "] / 2 + 1 = " + std::to_string(r.fft_sizes[u] / 2 + 1), u);
  }
  p->n = r.n; p->f0_stride = r.f0_stride; p->y_stride = r.y_stride; p->fs = r.fs;
  p->nbit = r.nbit; p->frame_period = r.frame_period;
  p->coded = r.coded;
  const int n_sizes = (int)p->sizes.size();
  int rc = 0;
  if (r.coded) {
    p->tsp.resize(n_sizes);
    p->tap.resize(n_sizes);
    for (int g = 0; g < n_sizes; ++g) {
      if (codec_decode_sp_tables(ctx, r.fs, p->sizes[g], r.dims, &p->tsp[g])) {
        if (!r.per_utt) return fail(ctx->last_error);
        const int u = (int)(std::find(p->size.begin(), p->size.end(), g) - p->size.begin());
        return fail_u(ctx->last_error + " (number_of_dimensions = " + std::to_string(r.dims) + ", fft_sizes[" +
                      std::to_string(u) + "] = " + std::to_string(p->sizes[g]) + ")", u);
      }
      codec_decode_ap_tables(r.fs, p->sizes[g], &p->tap[g]);
    }
    p->dims = r.dims;
    p->n_ap = n_sizes ? p->tap[0].dims : 0;
    if (p->n_ap > 0 && !r.ap) return fail("coded_aperiodicity is NULL, but fs has GetNumberOfAperiodicities(fs) > 0 bands");
  }
  p->modify = r.f0_scale || r.spectral_ratio;
  if (p->modify)
    rc = modify_plan(ctx, who, r.n, r.fft_size, r.fs, r.f0_scale, r.spectral_ratio, &p->mod,
                     r.per_utt ? r.fft_sizes : nullptr);
  if (packed) {
    if (!rc) rc = packed_lengths(ctx, who, "f", "frames", r.f_offsets, r.n, 2, &p->f_len);
    if (!rc) rc = packed_lengths(ctx, who, "y", "samples", r.y_offsets, r.n, 2, &p->y_len);
    if (rc) return rc;
    p->f_off.assign(r.f_offsets, r.f_offsets + r.n + 1);
    p->y_off.assign(r.y_offsets, r.y_offsets + r.n + 1);
    // the strides of a padded batch of these utterances: the sizing of a pass's decode tables and nominal pulse room
    p->f0_stride = p->y_stride = 0;
    for (int u = 0; u < r.n; ++u) { p->f0_stride = imax(p->f0_stride, p->f_len[u]); p->y_stride = imax(p->y_stride, p->y_len[u]); }
  } else {
    if (!rc) rc = row_lengths(ctx, who, "f0", r.f0_lengths, r.n, r.f0_stride, 2, &p->f_len);
    if (!rc) rc = row_lengths(ctx, who, "y", r.y_lengths, r.n, r.y_stride, 2, &p->y_len);
    if (rc) return rc;
  }
  if (r.transform) p->fp.assign(r.fp, r.fp + r.n);
  // DC remover of each size (GetDCRemover, synthesis.cpp:319-333), host libm like the reference
  p->dc_remover.resize(n_sizes);
  for (int g = 0; g < n_sizes; ++g) {
    const int fft_size = p->sizes[g];
    std::vector<double> &dcr = p->dc_remover[g];
    dcr.resize(fft_size);
    double dc = 0.0;
    for (int i = 0; i < fft_size / 2; ++i) {
      dcr[i] = 0.5 - 0.5 * cos(2.0 * kPi * (i + 1.0) / (1.0 + fft_size));
      dcr[fft_size - i - 1] = dcr[i];
      dc += dcr[i] * 2.0;
    }
    for (int i = 0; i < fft_size / 2; ++i) { dcr[i] /= dc; dcr[fft_size - i - 1] = dcr[i]; }
  }
  return 0;
}

SynthesisSizing::SynthesisSizing(const Ctx *ctx, const SynthesisPlan &p, int max_y)
    : fft_size(p.fft_size), y_stride(p.y_stride), fs(p.fs) {
  // The coded call holds one chunk's decoded envelope and aperiodicity (16 B per row entry and frame) and the decode
  // tables of every size.
  size_t tables = 0;
  if (p.coded) {
    ArenaPlan tp;
    for (size_t g = 0; g < p.sizes.size(); ++g) {
      tp.add(p.tsp[g].idx.size() * 4); tp.add(p.tsp[g].frac.size() * 8); tp.add(p.tsp[g].weight.size() * 16);
      tp.add(p.tap[g].idx.size() * 4); tp.add(p.tap[g].frac.size() * 8);
    }
    tables = tp.total;
  }
  decoded_per_utt = p.coded ? (size_t)p.f0_stride * p.row * 16 : 0;
  decoded_per_frame = p.coded ? (size_t)p.row * 16 : 0;
  // A modified call also holds the stretch tables, and per utterance its factor, table index and scaled f0 row (the
  // 256-byte alignment of the two small arrays is in the 4096 below).
  if (p.coded && p.modify) {
    tables += p.mod.device_bytes(0);
    decoded_per_utt += (size_t)p.f0_stride * 8 + 12;
    decoded_per_frame += 8;
  }
  // A call of several sizes holds the DC removers of the others, and per utterance its size and list entry.
  for (size_t g = 1; g < p.sizes.size(); ++g) tables += ((size_t)p.sizes[g] * 8 + 255) & ~(size_t)255;
  if (p.sizes.size() > 1) decoded_per_utt += 8;
  budget = (double)ctx->scratch_budget - (double)tables;
  // Pulse arrays and responses are sized for 1200 pulses per second (f0 <= 1.2 kHz; the +64 covers the ends).
  nominal_cap = (int)((double)max_y / p.fs * 1200.0) + 64;
  max_draws = (size_t)max_y + 8;
}

// PassLayout's bytes per utterance, with the 256-byte alignment of its small arrays rounded up to 4096
size_t SynthesisSizing::per_utt(int cap) const {
  return (size_t)y_stride * 16 + (size_t)cap * (4 + 8 + 8) + (size_t)cap * fft_size * 8 + 4096 + decoded_per_utt;
}

int SynthesisSizing::fit(int cap) const { return (int)dmin(65535.0, budget / (double)per_utt(cap)); }

int SynthesisSizing::cap_of(int y_len) const { return (int)((double)y_len / fs * 1200.0) + 64; }

// PassLayout's bytes of one utterance in a packed pass: phase and vuv, cap pulse slots (index, shift, draw count and
// offset) with their responses, its decoded rows, and 128 bytes for its entries of the small arrays (lengths, counts,
// offsets, factors, size lists)
size_t SynthesisSizing::packed_utt(int y_len, int f_len, int cap) const {
  return (size_t)y_len * 16 + (size_t)cap * (4 + 8 + 8 + (size_t)fft_size * 8) + (size_t)f_len * decoded_per_frame +
         128;
}

// the 256-byte alignment of a packed pass's sub-blocks
size_t SynthesisSizing::packed_pass() const { return (size_t)64 * 256; }

namespace {
// The scratch block of one pass of n utterances with room for cap pulses each.  Per size g: its DC remover and (coded)
// its decode tables.
// A padded pass gives every utterance y_stride samples, cap pulse slots and f0_stride frames; a packed pass gives each
// its own, back to back: the pass's totals are samples, pulses and frames, and it also holds the [n + 1] frame, sample
// and pulse offsets and the [n + G] per-group prefixes of pulses and frames.
struct PassLayout {
  size_t len, phase, vuv, pidx, psh, np, cnt, dcnt, doff, dtot, pl, resp;
  std::vector<size_t> dcr, sidx, sfrac, sw, aidx, afrac;
  size_t dsp = 0, dap = 0;   // coded
  size_t mod = 0, f0m = 0, fp = 0, fft_u = 0, list = 0, total;
  size_t offs = 0, cums = 0;   // packed
  PassLayout(const SynthesisPlan &p, int n, int cap)
      : PassLayout(p, n, (size_t)n * p.y_stride, (size_t)n * cap, (size_t)n * p.f0_stride, false) {}
  PassLayout(const SynthesisPlan &p, int n, size_t samples, size_t pulses, size_t frames, bool packed) {
    const size_t N = n, G = p.sizes.size();
    ArenaPlan a;
    len = a.add(2 * N * 4);                                          // f0 lengths, then y lengths
    phase = a.add(samples * 8); vuv = a.add(samples * 8);
    pidx = a.add(pulses * 4); psh = a.add(pulses * 8);
    np = a.add(N * 4); cnt = a.add(N * 4);
    dcnt = a.add(pulses * 4); doff = a.add(pulses * 4);
    dtot = a.add(N * 4); pl = a.add(N * 4);
    resp = a.add(pulses * p.fft_size * 8);
    for (size_t g = 0; g < G; ++g) dcr.push_back(a.add((size_t)p.sizes[g] * 8));
    if (p.coded) {
      dsp = a.add(frames * p.row * 8); dap = a.add(frames * p.row * 8);
      for (size_t g = 0; g < G; ++g) {
        const CodecTables &ts = p.tsp[g], &ta = p.tap[g];
        sidx.push_back(a.add(ts.idx.size() * 4)); sfrac.push_back(a.add(ts.frac.size() * 8));
        sw.push_back(a.add(ts.weight.size() * 16));
        aidx.push_back(a.add(ta.idx.size() * 4)); afrac.push_back(a.add(ta.frac.size() * 8));
      }
      if (p.modify) {
        mod = a.add(p.mod.device_bytes(n));
        if (!p.mod.scale.empty()) f0m = a.add(frames * 8);
      }
    }
    if (!p.fp.empty()) fp = a.add(N * 8);
    if (G > 1) { fft_u = a.add(N * 4); list = a.add(N * 4); }
    if (packed) { offs = a.add(3 * (N + 1) * 8); cums = a.add(2 * (N + G) * 8); }
    total = a.total;
  }
};

int log2_of(int v) {
  int lg = 0;
  while ((1 << lg) < v) ++lg;
  return lg;
}

// syn_pulse_kernel's dynamic shared memory at one fft_size
size_t pulse_smem(int fft_size) {
  const int half = fft_size / 2;
  return (size_t)(2 * fft_size + 2 * (half + 2) + (fft_size + 2) + 2 * (half + 1) + fft_size + WB_RED_DOUBLES) * 8;
}
}  // namespace

// nbit 0 writes the waveform (double), nbit 16 its 16-bit PCM (short).
int synthesis_run(Ctx *ctx, const SynthesisPlan &plan, int u0, int m, const SynthesisRows &rows) {
  if (m == 0) return 0;
  const int *f_len = plan.f_len.data() + u0, *y_len = plan.y_len.data() + u0;
  const int f0_stride = plan.f0_stride, y_stride = plan.y_stride, n_sizes = (int)plan.sizes.size();
  const size_t row = plan.row;
  const bool mixed = n_sizes > 1, packed = plan.packed();
  // packed: the offsets of this run's utterances, and where utterance v's rows and samples start from the run's first
  const long long *fo = packed ? plan.f_off.data() + u0 : nullptr, *yo = packed ? plan.y_off.data() + u0 : nullptr;
  auto frame_at = [&](int v) { return packed ? (size_t)(fo[v] - fo[0]) : (size_t)v * f0_stride; };
  auto sample_at = [&](int v) { return packed ? (size_t)(yo[v] - yo[0]) : (size_t)v * y_stride; };
  int max_y = 0;
  for (int i = 0; i < m; ++i) max_y = imax(max_y, y_len[i]);
  // The caller's f0 may be anything up to fs/2 (a pitch-shifted contour), so syn_timebase_kernel also counts the
  // pulses it could not store; a chunk where that count exceeds the cap is laid out again with room for its largest
  // count, in as many passes as the scratch budget needs.  The common case pays one read-back of n counts per chunk.
  // Every response slot holds the call's largest fft_size, so a pass's layout does not depend on which sizes it has.
  // A packed pass is a run of consecutive utterances whose own scratch fits the budget, each with room for its own
  // pulses; an utterance with more pulses than that gets room for exactly its count, and the pass is cut short until it
  // fits again.
  const SynthesisSizing sz(ctx, plan, max_y);
  const unsigned *table = rng_table_reserve(ctx, sz.max_draws);
  if (!table) return WORLD_B200_ENOMEM;
  const ModifyPlan *mod = plan.coded && plan.modify ? &plan.mod : nullptr;
  const bool scale_f0 = mod && !mod->scale.empty(), stretch = mod && !mod->table.empty();
  const int nominal_cap = sz.nominal_cap;
  auto fit = [&](int cap) { return sz.fit(cap); };
  const int chunk = packed ? 0 : balanced_chunk(imin(m, 65535), fit(nominal_cap));
  // packed: caps[i] is the pulse room of the pass's utterance i; the longest prefix of [v0, v0 + k) that fits
  std::vector<int> caps;
  auto packed_fit = [&](int v0, int k) {
    double bytes = (double)sz.packed_pass();
    int n = 0;
    while (n < k && n < 65535) {
      const int v = v0 + n;
      bytes += (double)sz.packed_utt(y_len[v], f_len[v], caps[n]);
      if (n > 0 && bytes > sz.budget) break;
      ++n;
    }
    return n;
  };
  auto packed_pass = [&](int v0) {
    caps.resize(m - v0);
    for (int i = 0; i < m - v0; ++i) caps[i] = sz.cap_of(y_len[v0 + i]);
    return packed_fit(v0, m - v0);
  };
#ifndef WB_EMU
  const int smem = (int)pulse_smem(plan.fft_size);
  cudaFuncSetAttribute(syn_pulse_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(syn_pulse_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
#endif
  std::vector<int> counts;
  int v0 = 0, n = packed ? packed_pass(0) : imin(chunk, m), pulse_cap = nominal_cap;   // this pass: [u0 + v0, +n)
  bool relaid = false;
  while (v0 < m) {
    // packed: the pass's offsets from its first utterance -- frames, samples, pulse slots
    std::vector<long long> offs(packed ? 3 * ((size_t)n + 1) : 0);
    long long *foff = offs.data(), *soff = foff + n + 1, *poff = soff + n + 1;
    size_t samples = 0, pulses = 0, frames = 0;
    if (packed) {
      for (int i = 0; i <= n; ++i) {
        foff[i] = (long long)(frame_at(v0 + i) - frame_at(v0));
        soff[i] = (long long)(sample_at(v0 + i) - sample_at(v0));
        poff[i] = i ? poff[i - 1] + caps[i - 1] : 0;
      }
      samples = soff[n]; pulses = poff[n]; frames = foff[n];
    }
    const PassLayout l = packed ? PassLayout(plan, n, samples, pulses, frames, true) : PassLayout(plan, n, pulse_cap);
    unsigned char *blk = arena_block(ctx, l.total);
    if (!blk) return WORLD_B200_ENOMEM;
    std::vector<int> l2((size_t)2 * n), pl(n, pulse_cap);
    if (packed) std::copy(caps.begin(), caps.begin() + n, pl.begin());
    int max_f = 0;
    for (int i = 0; i < n; ++i) { l2[i] = f_len[v0 + i]; l2[n + i] = y_len[v0 + i]; max_f = imax(max_f, l2[i]); }
    // the pass's utterances grouped by size: group g is list[first[g] .. first[g + 1])
    std::vector<int> fft_u(n), list, first(n_sizes + 1, 0);
    for (int g = 0; g < n_sizes; ++g) {
      first[g] = (int)list.size();
      for (int i = 0; i < n; ++i)
        if (plan.size[u0 + v0 + i] == g) { list.push_back(i); fft_u[i] = plan.sizes[g]; }
    }
    first[n_sizes] = n;
    int rc = dev_memcpy_h2d(ctx, blk + l.len, l2.data(), l2.size() * 4);
    for (int g = 0; g < n_sizes && !rc; ++g)
      rc = dev_memcpy_h2d(ctx, blk + l.dcr[g], plan.dc_remover[g].data(), (size_t)plan.sizes[g] * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + l.pl, pl.data(), (size_t)n * 4);
    if (!rc && !plan.fp.empty()) rc = dev_memcpy_h2d(ctx, blk + l.fp, plan.fp.data() + u0 + v0, (size_t)n * 8);
    if (!rc && mixed) rc = dev_memcpy_h2d(ctx, blk + l.fft_u, fft_u.data(), (size_t)n * 4);
    if (!rc && mixed) rc = dev_memcpy_h2d(ctx, blk + l.list, list.data(), (size_t)n * 4);
    if (!rc && packed) rc = dev_memcpy_h2d(ctx, blk + l.offs, offs.data(), offs.size() * 8);
    for (int g = 0; g < n_sizes && plan.coded; ++g) {
      const CodecTables &s = plan.tsp[g], &a = plan.tap[g];
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + l.sidx[g], s.idx.data(), s.idx.size() * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + l.sfrac[g], s.frac.data(), s.frac.size() * 8);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + l.sw[g], s.weight.data(), s.weight.size() * 16);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + l.aidx[g], a.idx.data(), a.idx.size() * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + l.afrac[g], a.frac.data(), a.frac.size() * 8);
    }
    ModifyDevice md = {};
    if (mod && !rc) rc = modify_upload(ctx, *mod, u0 + v0, n, blk + l.mod, &md);
    if (rc) return rc;
    const long long *d_off = packed ? (const long long *)(blk + l.offs) : nullptr;
    SynParams p{};
    p.f0 = rows.f0 + frame_at(v0); p.f_len = (const int *)(blk + l.len); p.f_stride = f0_stride;
    if (plan.coded) {
      p.sp = (const double *)(blk + l.dsp); p.ap = (const double *)(blk + l.dap);
    } else {
      p.sp = rows.sp + frame_at(v0) * row; p.ap = rows.ap + frame_at(v0) * row;
    }
    p.fft_size = plan.fft_size; p.lg_fft = log2_of(plan.fft_size); p.row = (int)row;
    p.fft_u = mixed ? (const int *)(blk + l.fft_u) : nullptr; p.list = nullptr;
    p.frame_period = plan.frame_period / 1000.0; p.fs = plan.fs;
    p.fp_u = plan.fp.empty() ? nullptr : (const double *)(blk + l.fp);
    p.y_len = (const int *)(blk + l.len) + n; p.y_stride = y_stride;
    p.phase = (double *)(blk + l.phase); p.vuv = (double *)(blk + l.vuv); p.flag_cnt = nullptr;
    p.pulse_idx = (int *)(blk + l.pidx); p.pulse_shift = (double *)(blk + l.psh); p.n_pulses = (int *)(blk + l.np);
    p.pulse_cap = pulse_cap; p.pulse_count = (int *)(blk + l.cnt);
    p.draw_cnt = (unsigned *)(blk + l.dcnt); p.draw_off = (unsigned *)(blk + l.doff);
    p.draw_tot = (unsigned *)(blk + l.dtot);
    p.draws = table;
    p.resp = (double *)(blk + l.resp); p.resp_n = plan.fft_size; p.dc_remover = (const double *)(blk + l.dcr[0]);
    p.y = plan.nbit ? nullptr : (double *)rows.y + sample_at(v0);
    p.y16 = plan.nbit ? (short *)rows.y + sample_at(v0) : nullptr;
    p.tw = ctx->twiddle;
    if (packed) {
      p.f_off = d_off; p.s_off = d_off + (n + 1); p.p_off = d_off + 2 * (n + 1);
      p.n_utts = n;
    }
    // a pass laid out from the counts reports a pulse beyond its arrays as a scratch overflow (status bit 4)
    p.status = relaid ? ctx->status_dev : nullptr;
    if (scale_f0) {
      // the time base, the pulse count (and the relaid pass it may call for) and the pulses all see the scaled contour
      double *f0m = (double *)(blk + l.f0m);
      modify_f0_launch(ctx, md, p.f_len, n, f0_stride, max_f, p.f0, f0m, p.f_off);
      p.f0 = f0m;
    }
    if (packed)
      WB_LAUNCH_COOP(syn_timebase_kernel<true>, dim3((unsigned)n), 256, 0, ctx->stream, p);
    else
      WB_LAUNCH_COOP(syn_timebase_kernel<false>, dim3((unsigned)n), 256, 0, ctx->stream, p);
    if (!relaid) {
      counts.resize(n);
      rc = dev_memcpy_d2h(ctx, counts.data(), p.pulse_count, (size_t)n * 4);
      if (!rc) rc = dev_sync(ctx);
      if (rc) return rc;
      int most = 0;
      bool over = false;
      for (int i = 0; i < n; ++i) {
        most = imax(most, counts[i]);
        if (packed && counts[i] > caps[i]) { caps[i] = counts[i]; over = true; }
      }
      if (packed ? over : most > pulse_cap) {
        // the time base is deterministic: run again over the first n' of these utterances, it finds the same pulses
        if (packed) {
          n = imax(1, packed_fit(v0, n));
        } else {
          pulse_cap = most;
          n = imin(n, imax(1, fit(pulse_cap)));
        }
        relaid = true;
        continue;
      }
    }
    // size group g of this pass: its utterance count, and its list on the device (null: the whole pass)
    auto group_n = [&](int g) { return first[g + 1] - first[g]; };
    auto group_list = [&](int g) { return mixed ? (const int *)(blk + l.list) + first[g] : nullptr; };
    // packed: per size group, the prefix sums of its utterances' pulses and frames ([group_n + 1] at first[g] + g):
    // the pulse and decode kernels run one CTA per pulse or frame, not over the padded grid
    std::vector<long long> cums(packed ? 2 * ((size_t)n + n_sizes) : 0);
    long long *pcum = cums.data(), *fcum = pcum + (n + n_sizes);
    for (int g = 0; g < n_sizes && packed; ++g) {
      long long *pc = pcum + first[g] + g, *fc = fcum + first[g] + g;
      pc[0] = fc[0] = 0;
      for (int j = 0; j < group_n(g); ++j) {
        const int i = list.empty() ? j : list[first[g] + j];
        pc[j + 1] = pc[j] + imin(counts[i], caps[i]);
        fc[j + 1] = fc[j] + f_len[v0 + i];
      }
    }
    if (packed) rc = dev_memcpy_h2d(ctx, blk + l.cums, cums.data(), cums.size() * 8);
    if (rc) return rc;
    const long long *pcum_d = packed ? (const long long *)(blk + l.cums) : nullptr;
    const long long *fcum_d = packed ? pcum_d + (n + n_sizes) : nullptr;
    if (plan.coded) {
      // DecodeSpectralEnvelope / DecodeAperiodicity of this pass's utterances, frames [0, f0_length), each at its size
      // into rows of the call's largest bins
      double *dsp = (double *)(blk + l.dsp), *dap = (double *)(blk + l.dap);
      const double *csp = rows.sp + frame_at(v0) * plan.dims;
      const double *cap = plan.n_ap > 0 ? rows.ap + frame_at(v0) * plan.n_ap : dap;
      for (int g = 0; g < n_sizes; ++g) {
        const CodecDeviceTables ts = {(const int *)(blk + l.sidx[g]), (const double *)(blk + l.sfrac[g]),
                                      (const double2 *)(blk + l.sw[g])};
        if (packed)
          codec_decode_packed_launch(ctx, true, plan.tsp[g], ts, plan.sizes[g], p.f_len, p.f_off, group_list(g),
                                     group_n(g), fcum_d + first[g] + g, fcum[first[g] + g + group_n(g)], csp, dsp,
                                     (int)row);
        else
          codec_decode_launch(ctx, true, plan.tsp[g], ts, plan.sizes[g], p.f_len, group_n(g), f0_stride, max_f, csp,
                              dsp, group_list(g), (int)row);
      }
      if (stretch) modify_stretch_launch(ctx, md, (int)row, mod->bins, p.f_len, n, f0_stride, max_f, dsp, p.f_off);
      // below 12 kHz there are no bands: the kernel reads no coded value (its input pointer only has to be valid)
      for (int g = 0; g < n_sizes; ++g) {
        const CodecDeviceTables ta = {(const int *)(blk + l.aidx[g]), (const double *)(blk + l.afrac[g]), nullptr};
        if (packed)
          codec_decode_packed_launch(ctx, false, plan.tap[g], ta, plan.sizes[g], p.f_len, p.f_off, group_list(g),
                                     group_n(g), fcum_d + first[g] + g, fcum[first[g] + g + group_n(g)], cap, dap,
                                     (int)row);
        else
          codec_decode_launch(ctx, false, plan.tap[g], ta, plan.sizes[g], p.f_len, group_n(g), f0_stride, max_f, cap,
                              dap, group_list(g), (int)row);
      }
    }
    scan_counts(ctx, p.draw_cnt, (const int *)(blk + l.pl), pulse_cap, nullptr, p.draw_off, p.draw_tot, n, p.p_off);
    // one launch per size, each with its own shared memory (and so its own occupancy)
    for (int g = 0; g < n_sizes; ++g) {
      if (group_n(g) == 0) continue;
      SynParams q = p;
      q.fft_size = plan.sizes[g]; q.lg_fft = log2_of(q.fft_size);
      q.dc_remover = (const double *)(blk + l.dcr[g]); q.list = group_list(g);
      if (packed) {
        const long long total = pcum[first[g] + g + group_n(g)];
        if (total == 0) continue;
        q.cum = pcum_d + first[g] + g; q.list_n = group_n(g);
        WB_LAUNCH_COOP(syn_pulse_kernel<true>, dim3((unsigned)total), 128, pulse_smem(q.fft_size), ctx->stream, q);
      } else {
        WB_LAUNCH_COOP(syn_pulse_kernel<false>, dim3((unsigned)pulse_cap, (unsigned)group_n(g)), 128,
                       pulse_smem(q.fft_size), ctx->stream, q);
      }
    }
    const dim3 grid = packed ? dim3((unsigned)((samples + 255) / 256)) : dim3((unsigned)((max_y + 255) / 256), (unsigned)n);
    if (plan.nbit)
      WB_LAUNCH_FLAT(syn_overlap_kernel<short>, grid, 256, 0, ctx->stream, p);
    else
      WB_LAUNCH_FLAT(syn_overlap_kernel<double>, grid, 256, 0, ctx->stream, p);
    rc = dev_check(ctx, "synthesis");
    if (rc) return rc;
    v0 += n;
    n = packed ? (v0 < m ? packed_pass(v0) : 0) : imin(chunk, m - v0);
    pulse_cap = nominal_cap;
    relaid = false;
  }
  return 0;
}

}  // namespace wb

using namespace wb;

// world_b200_synthesis_batch and the three world_b200_synthesis_coded_batch*: one plan, one run over the whole batch
static int synthesis_batch(WorldB200 *h, const SynthesisRequest &r) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  SynthesisPlan plan;
  const int rc = synthesis_plan(&h->c, r, "Synthesis", &plan);
  return rc ? rc : synthesis_run(&h->c, plan, 0, r.n, {r.f0, r.sp, r.ap, r.y});
}

static int synthesis_coded_batch(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                                 const double *coded_spectral_envelope, int number_of_dimensions,
                                 const double *coded_aperiodicity, int fft_size, double frame_period, int fs,
                                 const int *y_lengths, int y_stride, void *y, int nbit,
                                 const double *f0_scale = nullptr, const double *spectral_ratio = nullptr) {
  SynthesisRequest r{f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, coded_aperiodicity, fft_size,
                     frame_period, fs, y_lengths, y_stride, y, nbit};
  r.coded = true; r.dims = number_of_dimensions; r.f0_scale = f0_scale; r.spectral_ratio = spectral_ratio;
  return synthesis_batch(h, r);
}

extern "C" int world_b200_synthesis_batch(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts,
                                          int f0_stride, const double *spectrogram, const double *aperiodicity,
                                          int fft_size, double frame_period, int fs, const int *y_lengths,
                                          int y_stride, double *y) {
  return synthesis_batch(h, {f0, f0_lengths, n_utts, f0_stride, spectrogram, aperiodicity, fft_size, frame_period, fs,
                             y_lengths, y_stride, y, 0});
}

extern "C" int world_b200_synthesis_coded_batch_modified(WorldB200 *h, const double *f0, const int *f0_lengths,
                                                         int n_utts, int f0_stride,
                                                         const double *coded_spectral_envelope,
                                                         int number_of_dimensions, const double *coded_aperiodicity,
                                                         int fft_size, double frame_period, int fs,
                                                         const int *y_lengths, int y_stride, const double *f0_scale,
                                                         const double *spectral_ratio, int nbit, void *y) {
  return synthesis_coded_batch(h, f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, number_of_dimensions,
                               coded_aperiodicity, fft_size, frame_period, fs, y_lengths, y_stride, y, nbit, f0_scale,
                               spectral_ratio);
}

extern "C" int world_b200_synthesis_coded_batch(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts,
                                                int f0_stride, const double *coded_spectral_envelope,
                                                int number_of_dimensions, const double *coded_aperiodicity,
                                                int fft_size, double frame_period, int fs, const int *y_lengths,
                                                int y_stride, double *y) {
  return synthesis_coded_batch(h, f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, number_of_dimensions,
                               coded_aperiodicity, fft_size, frame_period, fs, y_lengths, y_stride, y, 0);
}

extern "C" int world_b200_synthesis_coded_batch_pcm16(WorldB200 *h, const double *f0, const int *f0_lengths,
                                                      int n_utts, int f0_stride, const double *coded_spectral_envelope,
                                                      int number_of_dimensions, const double *coded_aperiodicity,
                                                      int fft_size, double frame_period, int fs, const int *y_lengths,
                                                      int y_stride, short *y) {
  return synthesis_coded_batch(h, f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, number_of_dimensions,
                               coded_aperiodicity, fft_size, frame_period, fs, y_lengths, y_stride, y, 16);
}

// world_b200_modify_batch (fft_sizes NULL: fft_size for every utterance, rows of fft_size / 2 + 1) and
// world_b200_modify_batch_options (utterance u at fft_sizes[u], rows of row_stride)
// world_b200_modify_packed: f_offsets (host, [n_utts + 1]) instead of f0_lengths / f0_stride, row_stride 0 = the largest
// fft_sizes[u] / 2 + 1
// cv (world_b200_modify_curves / _curves_packed): DEVICE curves in place of the factors (which are then null), checked
// by curves_check after the host checks
static int modify_batch(WorldB200 *h, double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                        double *spectrogram, int row_stride, int fft_size, const int *fft_sizes, bool per_utt, int fs,
                        const double *f0_scale, const double *spectral_ratio, const long long *f_offsets = nullptr,
                        bool packed = false, const ModifyCurves *cv = nullptr) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  const char *who = cv ? "modify_curves" : "modify";
  auto fail = [&](const std::string &what) {
    ctx->last_error = std::string(who) + ": " + what;
    return WORLD_B200_EINVAL;
  };
  const bool stretch = spectral_ratio || (cv && cv->ratio);
  if (packed || cv) {
    if (n_utts < 0) return fail("n_utts must be >= 0");
    if (n_utts == 0) return 0;
  }
  if (packed) {
    if (!f_offsets) return fail("f_offsets must be given");
  } else if (n_utts < 0 || f0_stride <= 0) {
    return fail("n_utts must be >= 0 and f0_stride > 0");
  }
  if (cv && ((cv->f0 && !f0) || (cv->ratio && !spectrogram)))
    return fail("f0_curve needs f0 rows and spectral_ratio_curve needs spectrogram rows");
  if ((f0_scale && !f0) || (spectral_ratio && !spectrogram))
    return fail("f0_scale needs f0 rows and spectral_ratio needs spectrogram rows");
  if (per_utt && stretch) {
    if (!fft_sizes) return fail("fft_sizes must be given");
    if (fs <= 0) return fail("fs must be > 0");
    if (packed && row_stride == 0)
      for (int u = 0; u < n_utts; ++u) row_stride = imax(row_stride, fft_sizes[u] / 2 + 1);
    for (int u = 0; u < n_utts; ++u) {
      const int f = fft_sizes[u], why = f < 16 || f > 4096 || (f & (f - 1)) ? 1 : row_stride < f / 2 + 1 ? 2 : 0;
      if (why == 1)
        return fail("fft_sizes[" + std::to_string(u) + "] = " + std::to_string(f) +
                    " is not a power of two in [16, 4096] (utterance " + std::to_string(u) + ")");
      if (why == 2)
        return fail("row_stride = " + std::to_string(row_stride) + " is smaller than fft_sizes[" + std::to_string(u) +
                    "] / 2 + 1 = " + std::to_string(f / 2 + 1) + " (utterance " + std::to_string(u) + ")");
    }
  }
  // a length of 0 is allowed here: the utterance's rows are left alone
  std::vector<int> lens;
  ModifyPlan plan;
  int rc = packed ? packed_lengths(ctx, who, "f", "frames", f_offsets, n_utts, 0, &lens)
                  : row_lengths(ctx, who, "f0", f0_lengths, n_utts, f0_stride, 0, &lens);
  if (cv) {
    const long long *off = packed ? f_offsets : nullptr;
    if (!rc) rc = curves_check(ctx, who, *cv, n_utts, lens.data(), f0_stride, off, fft_sizes);
    return rc ? rc : curves_run(ctx, *cv, n_utts, lens.data(), f0_stride, off, fft_sizes, fs, row_stride, f0,
                                spectrogram);
  }
  if (!rc) rc = modify_plan(ctx, "modify", n_utts, fft_size, fs, f0_scale, spectral_ratio, &plan,
                            per_utt ? fft_sizes : nullptr);
  return rc ? rc : modify_run(ctx, plan, 0, n_utts, lens.data(), f0_stride, per_utt ? row_stride : plan.bins, f0,
                              spectrogram, packed ? f_offsets : nullptr);
}

extern "C" int world_b200_modify_batch(WorldB200 *h, double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                                       double *spectrogram, int fft_size, int fs, const double *f0_scale,
                                       const double *spectral_ratio) {
  return modify_batch(h, f0, f0_lengths, n_utts, f0_stride, spectrogram, 0, fft_size, nullptr, false, fs, f0_scale,
                      spectral_ratio);
}

extern "C" int world_b200_modify_batch_options(WorldB200 *h, double *f0, const int *f0_lengths, int n_utts,
                                               int f0_stride, double *spectrogram, int row_stride,
                                               const int *fft_sizes, int fs, const double *f0_scale,
                                               const double *spectral_ratio) {
  return modify_batch(h, f0, f0_lengths, n_utts, f0_stride, spectrogram, row_stride, 0, fft_sizes, true, fs, f0_scale,
                      spectral_ratio);
}

extern "C" int world_b200_synthesis_batch_options(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts,
                                                  int f0_stride, const double *spectrogram,
                                                  const double *aperiodicity, int row_stride, const int *fft_sizes,
                                                  double frame_period, int fs, const int *y_lengths, int y_stride,
                                                  double *y) {
  SynthesisRequest r{f0, f0_lengths, n_utts, f0_stride, spectrogram, aperiodicity, 0, frame_period, fs, y_lengths,
                     y_stride, y, 0};
  r.per_utt = true; r.fft_sizes = fft_sizes; r.row_stride = row_stride;
  return synthesis_batch(h, r);
}

extern "C" int world_b200_synthesis_coded_batch_options(WorldB200 *h, const double *f0, const int *f0_lengths,
                                                        int n_utts, int f0_stride,
                                                        const double *coded_spectral_envelope,
                                                        int number_of_dimensions, const double *coded_aperiodicity,
                                                        const int *fft_sizes, double frame_period, int fs,
                                                        const int *y_lengths, int y_stride, const double *f0_scale,
                                                        const double *spectral_ratio, int nbit, void *y) {
  SynthesisRequest r{f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, coded_aperiodicity, 0, frame_period,
                     fs, y_lengths, y_stride, y, nbit};
  r.coded = true; r.dims = number_of_dimensions; r.f0_scale = f0_scale; r.spectral_ratio = spectral_ratio;
  r.per_utt = true; r.fft_sizes = fft_sizes;
  return synthesis_batch(h, r);
}

// ---- packed rows: utterance u is frames [f_offsets[u], f_offsets[u + 1]) and samples [y_offsets[u], y_offsets[u + 1])
static int packed_missing(WorldB200 *h) {
  h->c.last_error = "Synthesis: f_offsets and y_offsets must be given";
  return WORLD_B200_EINVAL;
}

extern "C" int world_b200_synthesis_packed(WorldB200 *h, const double *f0, int n_utts, const long long *f_offsets,
                                           const double *spectrogram, const double *aperiodicity, int row_stride,
                                           const int *fft_sizes, double frame_period, int fs,
                                           const long long *y_offsets, double *y) {
  if (h && n_utts == 0) return 0;
  if (h && (!f_offsets || !y_offsets)) return packed_missing(h);
  SynthesisRequest r{f0, nullptr, n_utts, 0, spectrogram, aperiodicity, 0, frame_period, fs, nullptr, 0, y, 0};
  r.per_utt = true; r.fft_sizes = fft_sizes; r.row_stride = row_stride;
  r.f_offsets = f_offsets; r.y_offsets = y_offsets;
  return synthesis_batch(h, r);
}

extern "C" int world_b200_synthesis_coded_packed(WorldB200 *h, const double *f0, int n_utts,
                                                 const long long *f_offsets, const double *coded_spectral_envelope,
                                                 int number_of_dimensions, const double *coded_aperiodicity,
                                                 const int *fft_sizes, double frame_period, int fs,
                                                 const long long *y_offsets, const double *f0_scale,
                                                 const double *spectral_ratio, int nbit, void *y) {
  if (h && n_utts == 0) return 0;
  if (h && (!f_offsets || !y_offsets)) return packed_missing(h);
  SynthesisRequest r{f0, nullptr, n_utts, 0, coded_spectral_envelope, coded_aperiodicity, 0, frame_period, fs, nullptr,
                     0, y, nbit};
  r.coded = true; r.dims = number_of_dimensions; r.f0_scale = f0_scale; r.spectral_ratio = spectral_ratio;
  r.per_utt = true; r.fft_sizes = fft_sizes;
  r.f_offsets = f_offsets; r.y_offsets = y_offsets;
  return synthesis_batch(h, r);
}

extern "C" int world_b200_modify_packed(WorldB200 *h, double *f0, int n_utts, const long long *f_offsets,
                                        double *spectrogram, int row_stride, const int *fft_sizes, int fs,
                                        const double *f0_scale, const double *spectral_ratio) {
  return modify_batch(h, f0, nullptr, n_utts, 0, spectrogram, row_stride, 0, fft_sizes, true, fs, f0_scale,
                      spectral_ratio, f_offsets, true);
}

extern "C" int world_b200_modify_curves(WorldB200 *h, double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                                        double *spectrogram, int row_stride, const int *fft_sizes, int fs,
                                        const double *f0_curve, const double *spectral_ratio_curve) {
  ModifyCurves cv;
  cv.f0 = f0_curve; cv.ratio = spectral_ratio_curve;
  return modify_batch(h, f0, f0_lengths, n_utts, f0_stride, spectrogram, row_stride, 0, fft_sizes, true, fs, nullptr,
                      nullptr, nullptr, false, &cv);
}

extern "C" int world_b200_modify_curves_packed(WorldB200 *h, double *f0, int n_utts, const long long *f_offsets,
                                               double *spectrogram, int row_stride, const int *fft_sizes, int fs,
                                               const double *f0_curve, const double *spectral_ratio_curve) {
  ModifyCurves cv;
  cv.f0 = f0_curve; cv.ratio = spectral_ratio_curve;
  return modify_batch(h, f0, nullptr, n_utts, 0, spectrogram, row_stride, 0, fft_sizes, true, fs, nullptr, nullptr,
                      f_offsets, true, &cv);
}
