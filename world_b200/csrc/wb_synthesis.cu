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
//                         inverse transforms, DC removal -> one response of fft_size samples
//   syn_overlap_kernel    output sample -> thread: sums the responses covering it in pulse order
//                         (the reference's accumulation order, so the sum is deterministic)
// FFT conventions (SURVEY.md App. A0): c2c FORWARD of a == FFT(conj a); c2r of X == Re FFT(conj X~)
// with X~ the Hermitian extension -- both are forward transforms of wb_fft.cuh.
#include "wb_internal.h"
#include "wb_spectral.cuh"
#include "../../include/world_b200.h"
#include <type_traits>
#include <vector>

namespace wb {

struct SynParams {
  const double *f0; const int *f_len; int f_stride;
  const double *sp; const double *ap; int fft_size, lg_fft;
  double frame_period;      // seconds
  int fs;
  const int *y_len; int y_stride;
  // time base scratch
  double *phase;            // [n][y_stride] running phase, then wrapped phase
  double *vuv;              // [n][y_stride] interpolated vuv (0/1)
  int *flag_cnt;            // [n][258]
  int *pulse_idx; double *pulse_shift; int *n_pulses; int pulse_cap;   // [n][pulse_cap]
  int *pulse_count;         // [n] pulses found, also those beyond pulse_cap (the host sizes the arrays from it)
  unsigned *draw_cnt; unsigned *draw_off; unsigned *draw_tot;
  const unsigned *draws; size_t draw_stride;
  double *resp;             // [n][pulse_cap][fft_size]
  const double *dc_remover; // [fft_size]
  double *y;
  const double2 *tw;
  int *status;
  short *y16;               // [n][y_stride] 16-bit PCM output (syn_overlap_kernel<short>), else null
};

WB_KERNEL(256, 2) syn_timebase_kernel(SynParams p) {
  WB_SHARED int cnt[258];
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int L = p.f_len[u], n = p.y_len[u], fs = p.fs;
  const double fp = p.frame_period;
  const double lowest_f0 = fs / p.fft_size + 1.0;   // synthesis.cpp:362 (integer division, then + 1.0)
  const double *f0 = p.f0 + (size_t)u * p.f_stride;
  double *phase = p.phase + (size_t)u * p.y_stride;
  double *vuv = p.vuv + (size_t)u * p.y_stride;
  int *pidx = p.pulse_idx + (size_t)u * p.pulse_cap;
  double *pshift = p.pulse_shift + (size_t)u * p.pulse_cap;
  unsigned *dcnt = p.draw_cnt + (size_t)u * p.pulse_cap;
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
    p.n_pulses[u] = imin(run, p.pulse_cap);
    p.pulse_count[u] = run;   // run > pulse_cap: the host lays the chunk out again before anything reads the list
    if (run > p.pulse_cap) atomicOr_status(p.status, 4);   // status is null unless the counts sized this layout
  }
  WB_SYNC();
  int k = cnt[tid];
  for (int i = lo; i < hi; ++i) {
    if (fabs(phase[i + 1] - phase[i]) > kPi) {
      if (k < p.pulse_cap) {
        pidx[k] = i;
        const double y1 = phase[i] - 2.0 * kPi, y2 = phase[i + 1];
        pshift[k] = (-y1 / (y2 - y1)) / fs;
      }
      ++k;
    }
  }
  WB_SYNC();
  // noise_size = idx[min(np-1, i+1)] - idx[i] draws per pulse (:372-374, :19-25)
  const int np = imin(cnt[nth], p.pulse_cap);
  for (int i = tid; i < p.pulse_cap; i += nth)
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

WB_KERNEL(128, 3) syn_pulse_kernel(SynParams p) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const int u = blockIdx.y, pi = blockIdx.x;
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
  const int idx = p.pulse_idx[(size_t)u * p.pulse_cap + pi];
  const int idx_next = p.pulse_idx[(size_t)u * p.pulse_cap + imin(np - 1, pi + 1)];
  const int noise_size = idx_next - idx;
  const double shift = p.pulse_shift[(size_t)u * p.pulse_cap + pi];
  const double current_vuv = p.vuv[(size_t)u * p.y_stride + idx];
  const double current_time = idx / static_cast<double>(fs);
  double *resp = p.resp + ((size_t)u * p.pulse_cap + pi) * N;
  const size_t bins = half + 1;
  const double *sp = p.sp + (size_t)u * p.f_stride * bins, *ap = p.ap + (size_t)u * p.f_stride * bins;

  // GetSpectralEnvelope / GetAperiodicRatio (:140-179)
  const int fl = imin(L - 1, static_cast<int>(floor(current_time / p.frame_period)));
  const int ce = imin(L - 1, static_cast<int>(ceil(current_time / p.frame_period)));
  const double interp = current_time / p.frame_period - fl;
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

  // ---- aperiodic response (:36-69)
  if (noise_size > 0) {
    const unsigned *draw = p.draws + (size_t)u * p.draw_stride + p.draw_off[(size_t)u * p.pulse_cap + pi];
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
  } else {
    // last pulse: noise_size = 0 -> zero noise, sqrt(0) kills the periodic part (:372-374)
    for (int i = tid; i < N; i += nth) resp[i] = 0.0;
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
template <typename Out>
WB_KERNEL_PLAIN syn_overlap_kernel(SynParams p) {
  const int u = blockIdx.y;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = p.y_len[u];
  if (s >= n) return;
  const int N = p.fft_size, half = N / 2, np = p.n_pulses[u];
  const int *pidx = p.pulse_idx + (size_t)u * p.pulse_cap;
  // pulse i covers samples idx_i - half + 1 .. idx_i + half  ->  idx_i in [s - half, s + half - 1]
  int lo = 0, hi = np;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (pidx[mid] < s - half) lo = mid + 1; else hi = mid; }
  double acc = 0.0;
  for (int i = lo; i < np && pidx[i] <= s + half - 1; ++i) {
    const int j = s - (pidx[i] - half + 1);
    acc += p.resp[((size_t)u * p.pulse_cap + i) * N + j];
  }
  if constexpr (std::is_same<Out, short>::value) p.y16[(size_t)u * p.y_stride + s] = pcm16_of(acc);
  else p.y[(size_t)u * p.y_stride + s] = acc;
}

int synthesis_fft(Ctx *ctx, int fft_size, int *lg_out) {
  int lg = 0;
  while ((1 << lg) < fft_size) ++lg;
  if ((1 << lg) != fft_size || fft_size < 16 || fft_size > WB_TW_N / 2) {
    ctx->last_error = "Synthesis: fft_size must be a power of two in [16, 4096]";
    return WORLD_B200_EINVAL;
  }
  *lg_out = lg;
  return 0;
}

int synthesis_coded_tables(Ctx *ctx, int fs, int fft_size, int number_of_dimensions, bool have_aperiodicity,
                           CodedRows *coded) {
  const int rc = codec_decode_sp_tables(ctx, fs, fft_size, number_of_dimensions, &coded->tsp);
  if (rc) return rc;
  codec_decode_ap_tables(fs, fft_size, &coded->tap);
  if (coded->tap.dims > 0 && !have_aperiodicity) {
    ctx->last_error = "Synthesis: coded_aperiodicity is NULL, but fs has GetNumberOfAperiodicities(fs) > 0 bands";
    return WORLD_B200_EINVAL;
  }
  return 0;
}

int synthesis_lengths(Ctx *ctx, const int *f0_lengths, int n_utts, int f0_stride, const int *y_lengths, int y_stride,
                      int *lens) {
  for (int i = 0; i < n_utts; ++i) {
    lens[i] = f0_lengths ? f0_lengths[i] : f0_stride;
    lens[n_utts + i] = y_lengths ? y_lengths[i] : y_stride;
    if (lens[i] < 2 || lens[i] > f0_stride || lens[n_utts + i] < 2 || lens[n_utts + i] > y_stride) {
      ctx->last_error = "Synthesis: lengths outside the padded rows (need f0_length >= 2, y_length >= 2)";
      return WORLD_B200_EINVAL;
    }
  }
  return 0;
}

SynthesisSizing::SynthesisSizing(const Ctx *ctx, const CodedRows *coded, int fft_size, int f0_stride, int y_stride,
                                 int max_y, int fs)
    : fft_size(fft_size), y_stride(y_stride) {
  const size_t bins = (size_t)fft_size / 2 + 1;
  // The coded call holds one chunk's decoded envelope and aperiodicity (16 B per bin and frame) and the decode tables.
  size_t tables = 0;
  if (coded) {
    ArenaPlan tp;
    tp.add(coded->tsp.idx.size() * 4); tp.add(coded->tsp.frac.size() * 8); tp.add(coded->tsp.weight.size() * 16);
    tp.add(coded->tap.idx.size() * 4); tp.add(coded->tap.frac.size() * 8);
    tables = tp.total;
  }
  decoded_per_utt = coded ? (size_t)f0_stride * bins * 16 : 0;
  budget = (double)ctx->scratch_budget - (double)tables;
  // Pulse arrays and responses are sized for 1200 pulses per second (f0 <= 1.2 kHz; the +64 covers the ends).
  nominal_cap = (int)((double)max_y / fs * 1200.0) + 64;
  draw_stride = (size_t)max_y + 8;
}

size_t SynthesisSizing::per_utt(int cap) const {
  return (size_t)y_stride * 16 + (size_t)cap * (4 + 8 + 8) + (size_t)cap * fft_size * 8 + draw_stride * 4 + 4096 +
         decoded_per_utt;
}

int SynthesisSizing::fit(int cap) const { return (int)dmin(65535.0, budget / (double)per_utt(cap)); }

// The chunk driver of both entry points: full rows (spectrogram / aperiodicity) or, with `coded`, rows decoded per
// chunk into the chunk's block.  nbit 0 writes the waveform (double), nbit 16 its 16-bit PCM (short).
int synthesis_run(Ctx *ctx, const double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                  const double *spectrogram, const double *aperiodicity, const CodedRows *coded, int fft_size, int lg,
                  double frame_period, int fs, const int *y_lengths, int y_stride, void *y, int nbit) {
  if (n_utts == 0) return 0;
  std::vector<int> lens((size_t)2 * n_utts);
  int rc = synthesis_lengths(ctx, f0_lengths, n_utts, f0_stride, y_lengths, y_stride, lens.data());
  if (rc) return rc;
  int max_y = 0;
  for (int i = 0; i < n_utts; ++i) max_y = imax(max_y, lens[n_utts + i]);
  // DC remover (GetDCRemover, synthesis.cpp:319-333), host libm like the reference
  std::vector<double> dcr(fft_size);
  {
    double dc = 0.0;
    for (int i = 0; i < fft_size / 2; ++i) {
      dcr[i] = 0.5 - 0.5 * cos(2.0 * kPi * (i + 1.0) / (1.0 + fft_size));
      dcr[fft_size - i - 1] = dcr[i];
      dc += dcr[i] * 2.0;
    }
    for (int i = 0; i < fft_size / 2; ++i) { dcr[i] /= dc; dcr[fft_size - i - 1] = dcr[i]; }
  }
  const int half = fft_size / 2;
  const size_t bins = (size_t)half + 1;
  // The caller's f0 may be anything up to fs/2 (a pitch-shifted contour), so syn_timebase_kernel also counts the
  // pulses it could not store; a chunk where that count exceeds the cap is laid out again with room for its largest
  // count, in as many passes as the scratch budget needs.  The common case pays one read-back of n counts per chunk.
  const SynthesisSizing sz(ctx, coded, fft_size, f0_stride, y_stride, max_y, fs);
  const int nominal_cap = sz.nominal_cap;
  const size_t draw_stride = sz.draw_stride;
  auto fit = [&](int cap) { return sz.fit(cap); };
  const int chunk = balanced_chunk(imin(n_utts, 65535), fit(nominal_cap));
  const size_t smem = (size_t)(2 * fft_size + 2 * (half + 2) + (fft_size + 2) + 2 * (half + 1) + fft_size + WB_RED_DOUBLES) * 8;
#ifndef WB_EMU
  cudaFuncSetAttribute(syn_pulse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  std::vector<int> counts;
  int u0 = 0, n = imin(chunk, n_utts), pulse_cap = nominal_cap;
  bool relaid = false;
  while (u0 < n_utts) {
    ArenaPlan plan;
    const size_t o_len = plan.add((size_t)2 * n * 4);
    const size_t o_phase = plan.add((size_t)n * y_stride * 8), o_vuv = plan.add((size_t)n * y_stride * 8);
    const size_t o_pidx = plan.add((size_t)n * pulse_cap * 4), o_psh = plan.add((size_t)n * pulse_cap * 8);
    const size_t o_np = plan.add((size_t)n * 4), o_cnt = plan.add((size_t)n * 4);
    const size_t o_dc = plan.add((size_t)n * pulse_cap * 4), o_do = plan.add((size_t)n * pulse_cap * 4);
    const size_t o_dt = plan.add((size_t)n * 4), o_pl = plan.add((size_t)n * 4);
    const size_t o_draws = plan.add((size_t)n * draw_stride * 4);
    const size_t o_resp = plan.add((size_t)n * pulse_cap * fft_size * 8);
    const size_t o_dcr = plan.add((size_t)fft_size * 8);
    size_t o_dsp = 0, o_dap = 0, o_sidx = 0, o_sfrac = 0, o_sw = 0, o_aidx = 0, o_afrac = 0;
    if (coded) {
      o_dsp = plan.add((size_t)n * f0_stride * bins * 8); o_dap = plan.add((size_t)n * f0_stride * bins * 8);
      o_sidx = plan.add(coded->tsp.idx.size() * 4); o_sfrac = plan.add(coded->tsp.frac.size() * 8);
      o_sw = plan.add(coded->tsp.weight.size() * 16);
      o_aidx = plan.add(coded->tap.idx.size() * 4); o_afrac = plan.add(coded->tap.frac.size() * 8);
    }
    unsigned char *blk = arena_block(ctx, plan.total);
    if (!blk) return WORLD_B200_ENOMEM;
    std::vector<int> l2((size_t)2 * n), pl(n, pulse_cap);
    for (int i = 0; i < n; ++i) { l2[i] = lens[u0 + i]; l2[n + i] = lens[n_utts + u0 + i]; }
    rc = dev_memcpy_h2d(ctx, blk + o_len, l2.data(), l2.size() * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_dcr, dcr.data(), dcr.size() * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_pl, pl.data(), (size_t)n * 4);
    if (coded) {
      const CodecTables &s = coded->tsp, &a = coded->tap;
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_sidx, s.idx.data(), s.idx.size() * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_sfrac, s.frac.data(), s.frac.size() * 8);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_sw, s.weight.data(), s.weight.size() * 16);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_aidx, a.idx.data(), a.idx.size() * 4);
      if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_afrac, a.frac.data(), a.frac.size() * 8);
    }
    if (rc) return rc;
    SynParams p;
    p.f0 = f0 + (size_t)u0 * f0_stride; p.f_len = (const int *)(blk + o_len); p.f_stride = f0_stride;
    if (coded) {
      p.sp = (const double *)(blk + o_dsp); p.ap = (const double *)(blk + o_dap);
    } else {
      p.sp = spectrogram + (size_t)u0 * f0_stride * bins; p.ap = aperiodicity + (size_t)u0 * f0_stride * bins;
    }
    p.fft_size = fft_size; p.lg_fft = lg; p.frame_period = frame_period / 1000.0; p.fs = fs;
    p.y_len = (const int *)(blk + o_len) + n; p.y_stride = y_stride;
    p.phase = (double *)(blk + o_phase); p.vuv = (double *)(blk + o_vuv); p.flag_cnt = nullptr;
    p.pulse_idx = (int *)(blk + o_pidx); p.pulse_shift = (double *)(blk + o_psh); p.n_pulses = (int *)(blk + o_np);
    p.pulse_cap = pulse_cap; p.pulse_count = (int *)(blk + o_cnt);
    p.draw_cnt = (unsigned *)(blk + o_dc); p.draw_off = (unsigned *)(blk + o_do); p.draw_tot = (unsigned *)(blk + o_dt);
    p.draws = (const unsigned *)(blk + o_draws); p.draw_stride = draw_stride;
    p.resp = (double *)(blk + o_resp); p.dc_remover = (const double *)(blk + o_dcr);
    p.y = nbit ? nullptr : (double *)y + (size_t)u0 * y_stride;
    p.y16 = nbit ? (short *)y + (size_t)u0 * y_stride : nullptr;
    p.tw = ctx->twiddle;
    // a pass laid out from the counts reports a pulse beyond its arrays as a scratch overflow (status bit 4)
    p.status = relaid ? ctx->status_dev : nullptr;
    WB_LAUNCH_COOP(syn_timebase_kernel, dim3((unsigned)n), 256, 0, ctx->stream, p);
    if (!relaid) {
      counts.resize(n);
      rc = dev_memcpy_d2h(ctx, counts.data(), p.pulse_count, (size_t)n * 4);
      if (!rc) rc = dev_sync(ctx);
      if (rc) return rc;
      int most = 0;
      for (int i = 0; i < n; ++i) most = imax(most, counts[i]);
      if (most > pulse_cap) {
        // the time base is deterministic: run again over the first n' of these utterances, it finds the same pulses
        pulse_cap = most;
        n = imin(n, imax(1, fit(pulse_cap)));
        relaid = true;
        continue;
      }
    }
    if (coded) {
      // DecodeSpectralEnvelope / DecodeAperiodicity of this pass's utterances, frames [0, f0_length)
      int max_f = 0;
      for (int i = 0; i < n; ++i) max_f = imax(max_f, l2[i]);
      const CodecDeviceTables ts = {(const int *)(blk + o_sidx), (const double *)(blk + o_sfrac),
                                    (const double2 *)(blk + o_sw)};
      const CodecDeviceTables ta = {(const int *)(blk + o_aidx), (const double *)(blk + o_afrac), nullptr};
      double *dsp = (double *)(blk + o_dsp), *dap = (double *)(blk + o_dap);
      codec_decode_launch(ctx, true, coded->tsp, ts, fft_size, p.f_len, n, f0_stride, max_f,
                          coded->sp + (size_t)u0 * f0_stride * coded->tsp.dims, dsp);
      // below 12 kHz there are no bands: the kernel reads no coded value (its input pointer only has to be valid)
      codec_decode_launch(ctx, false, coded->tap, ta, fft_size, p.f_len, n, f0_stride, max_f,
                          coded->ap ? coded->ap + (size_t)u0 * f0_stride * coded->tap.dims : dap, dap);
    }
    scan_counts(ctx, p.draw_cnt, (const int *)(blk + o_pl), pulse_cap, nullptr, p.draw_off, p.draw_tot, n);
    rng_fill(ctx, p.draw_tot, (unsigned *)(blk + o_draws), draw_stride, draw_stride, n);
    WB_LAUNCH_COOP(syn_pulse_kernel, dim3((unsigned)pulse_cap, (unsigned)n), 128, smem, ctx->stream, p);
    if (nbit)
      WB_LAUNCH_FLAT(syn_overlap_kernel<short>, dim3((unsigned)((max_y + 255) / 256), (unsigned)n), 256, 0, ctx->stream, p);
    else
      WB_LAUNCH_FLAT(syn_overlap_kernel<double>, dim3((unsigned)((max_y + 255) / 256), (unsigned)n), 256, 0, ctx->stream, p);
    rc = dev_check(ctx, "synthesis");
    if (rc) return rc;
    u0 += n;
    n = imin(chunk, n_utts - u0);
    pulse_cap = nominal_cap;
    relaid = false;
  }
  return 0;
}

}  // namespace wb

using namespace wb;

extern "C" int world_b200_synthesis_batch(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts,
                                          int f0_stride, const double *spectrogram, const double *aperiodicity,
                                          int fft_size, double frame_period, int fs, const int *y_lengths,
                                          int y_stride, double *y) {
  if (!h || !f0 || !spectrogram || !aperiodicity || !y || n_utts < 0 || fs <= 0 || frame_period <= 0)
    return WORLD_B200_EINVAL;
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  Ctx *ctx = reinterpret_cast<Ctx *>(h);
  int lg = 0;
  const int rc = synthesis_fft(ctx, fft_size, &lg);
  if (rc) return rc;
  return synthesis_run(ctx, f0, f0_lengths, n_utts, f0_stride, spectrogram, aperiodicity, nullptr, fft_size, lg,
                       frame_period, fs, y_lengths, y_stride, y, 0);
}

// world_b200_synthesis_coded_batch (nbit 0, y double) and world_b200_synthesis_coded_batch_pcm16 (nbit 16, y short)
static int synthesis_coded_batch(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                                 const double *coded_spectral_envelope, int number_of_dimensions,
                                 const double *coded_aperiodicity, int fft_size, double frame_period, int fs,
                                 const int *y_lengths, int y_stride, void *y, int nbit) {
  if (!h || !f0 || !coded_spectral_envelope || !y || n_utts < 0 || fs <= 0 || frame_period <= 0)
    return WORLD_B200_EINVAL;
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  Ctx *ctx = reinterpret_cast<Ctx *>(h);
  int lg = 0;
  int rc = synthesis_fft(ctx, fft_size, &lg);
  if (rc) return rc;
  CodedRows coded;
  rc = synthesis_coded_tables(ctx, fs, fft_size, number_of_dimensions, coded_aperiodicity != nullptr, &coded);
  if (rc) return rc;
  coded.sp = coded_spectral_envelope;
  coded.ap = coded.tap.dims > 0 ? coded_aperiodicity : nullptr;
  return synthesis_run(ctx, f0, f0_lengths, n_utts, f0_stride, nullptr, nullptr, &coded, fft_size, lg, frame_period,
                       fs, y_lengths, y_stride, y, nbit);
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
