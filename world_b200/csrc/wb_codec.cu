// wb_codec.cu -- batched codec and ingest (SURVEY.md 8 rows f2 and f3: the callers / data formats on
// either side of the analysis path).
//
// Replaces CodeSpectralEnvelope / DecodeSpectralEnvelope / CodeAperiodicity / DecodeAperiodicity
// (codec.cpp:221-324, helpers :22-211) and the sample conversion of wavread (tools/audioio.cpp:217-252).
//   code_sp_kernel    (utterance, frame) -> CTA: log of the envelope row, interpolation onto the mel
//                     grid (interp1 with host-made index / fraction tables: both axes are frame
//                     independent), DCT-II as one real FFT of fft_size/2 (DCTForCodec :73-89)
//   decode_sp_kernel  (utterance, frame) -> CTA: weighted cepstrum -> one complex FFT of fft_size/2
//                     (the reference's c2c BACKWARD is conj(FFT(a)), fft.cpp:36-46; only its real part
//                     is used), de-interleave, interpolation back to the linear axis, exp
//   code_ap_kernel    frame -> thread: dB value at 3 kHz multiples by interp1Q (:228-238)
//   decode_ap_kernel  (utterance, frame) -> CTA: V/UV test on the mean of the coded values (:29-41),
//                     interp1 over {0, 3k, ..., fs/2} and 10^(v/20) (:46-55)
//   pcm_kernel        sample -> thread: little-endian signed PCM -> sample / 2^(nbit-1)
// Host side: every axis, index table and DCT weight is computed with the reference's own double
// expressions and the host libm, so the interpolation indices are the reference's.
#include "wb_chain.h"
#include "../../include/world_b200.h"
#include <math.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>

namespace wb {

// constantnumbers.h:19,35-36,45-48
static const double kCodecFrequencyInterval = 3000.0;
static const double kCodecUpperLimit = 15000.0;
static const double kCodecM0 = 1127.01048;
static const double kCodecF0 = 700.0;
static const double kCodecFloorFrequency = 40.0;
static const double kCodecCeilFrequency = 20000.0;
static const double kCodecSafeGuardMinimum = 0.000000000001;

struct CodecParams {
  const int *f_len; int f_stride;
  const double *in; double *out;
  int bins;                   // fft_size / 2 + 1
  int dims;                   // coded values per frame
  int max_dim, lg;            // fft_size / 2 and its log2 (spectral envelope only)
  const int *idx;             // interpolation: left node of each target point
  const double *frac;         // interpolation: (xi - x[k-1]) / (x[k] - x[k-1])
  const double2 *weight;      // DCT / IDCT weights
  double norm;                // sqrt(fft_size / 2)
  const double2 *tw;
  const int *list;            // the utterance of each blockIdx.y, or NULL: blockIdx.y itself
  int row;                    // doubles per full frame row (>= bins): decode's output, code's input
  // packed rows (null: padded rows of f_stride): utterance u's frame i is row f_off[u] + i of in and out; a frame of
  // the launch (blockIdx.x, code_ap_kernel: its thread) is one of entry j of list, which owns frames [cum[j], cum[j + 1])
  const long long *f_off, *cum;
  int list_n;
};

// the utterance, frame and (in and out) row of this CTA
struct DecodeAt { int u, f; size_t row; };
WB_DEV DecodeAt decode_at(const CodecParams &p) {
  if (p.cum) {
    const int j = packed_find(p.cum, p.list_n, (long long)blockIdx.x);
    const int u = p.list ? p.list[j] : j, f = (int)(blockIdx.x - p.cum[j]);
    return {u, f, (size_t)p.f_off[u] + f};
  }
  const int u = p.list ? p.list[blockIdx.y] : blockIdx.y, f = blockIdx.x;
  return {u, f, (size_t)u * p.f_stride + f};
}

// kPacked: packed rows (p.cum), a compile-time choice so that the padded kernel keeps its own code
template <bool kPacked>
WB_KERNEL(128, 8) code_sp_kernel(CodecParams p) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const DecodeAt at = kPacked ? decode_at(p) : DecodeAt{(int)blockIdx.y, (int)blockIdx.x,
                                                        (size_t)blockIdx.y * p.f_stride + blockIdx.x};
  if (at.f >= p.f_len[at.u]) return;
  double *lgs = smem;                       // bins (+1 pad)
  double *buf = smem + ((p.bins + 2) & ~1); // max_dim + 2
  const double *row = p.in + at.row * p.row;
  for (int j = tid; j < p.bins; j += nth) lgs[j] = log(row[j]);                     // codec.cpp:288-289
  WB_SYNC();
  const int M = p.max_dim, bias = M / 2;
  for (int i = tid; i < bias; i += nth) {                                           // :77-81 on top of :121-122
    const int a = 2 * i, b = M - 2 * i - 1;
    const int ka = __ldg(p.idx + a), kb = __ldg(p.idx + b);
    buf[i] = lgs[ka] + __ldg(p.frac + a) * (lgs[ka + 1] - lgs[ka]);
    buf[i + bias] = lgs[kb] + __ldg(p.frac + b) * (lgs[kb + 1] - lgs[kb]);
  }
  WB_SYNC();
  rfft_forward(buf, p.lg, p.tw);
  const double2 *X = reinterpret_cast<const double2 *>(buf);
  // packed: the row is looked up again after the transform rather than held across it
  double *out = p.out + (kPacked ? decode_at(p).row : at.row) * p.dims;
  for (int d = tid; d < p.dims; d += nth) {                                         // :85-88
    const double2 w = __ldg(p.weight + d);
    out[d] = (X[d].x * w.x - X[d].y * w.y) / p.norm;
  }
}

WB_KERNEL(128, 8) decode_sp_kernel(CodecParams p) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const DecodeAt at = decode_at(p);
  if (at.f >= p.f_len[at.u]) return;
  const int M = p.max_dim;
  double2 *z = reinterpret_cast<double2 *>(smem);  // M complex
  double *mel = smem + 2 * M;                      // M + 2
  const double *c = p.in + at.row * p.dims;
  for (int d = tid; d < M; d += nth) {                                              // :97-107
    double2 v = make_double2(0.0, 0.0);
    if (d < p.dims) {
      const double2 w = __ldg(p.weight + d);
      v = make_double2(c[d] * w.x * p.norm, -c[d] * w.y * p.norm);
    }
    z[d] = v;
  }
  WB_SYNC();
  cfft_forward(z, p.lg, p.tw);
  for (int i = tid; i < M / 2; i += nth) {                                          // :111-115, :147-148
    mel[1 + 2 * i] = z[i].x;
    mel[2 + 2 * i] = z[M - i - 1].x;
  }
  WB_SYNC();
  if (tid == 0) { mel[0] = mel[1]; mel[M + 1] = mel[M]; }
  WB_SYNC();
  double *out = p.out + at.row * p.row;
  for (int j = tid; j < p.bins; j += nth) {                                         // :150-154
    const int k = __ldg(p.idx + j);
    const double v = mel[k] + __ldg(p.frac + j) * (mel[k + 1] - mel[k]);
    out[j] = exp(v / M);
  }
}

WB_KERNEL_PLAIN code_ap_kernel(CodecParams p) {
  size_t r;
  if (p.cum) {   // packed rows: the thread's frame of the launch
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= p.cum[p.list_n]) return;
    const int j = packed_find(p.cum, p.list_n, g);
    r = (size_t)(p.f_off[p.list ? p.list[j] : j] + (g - p.cum[j]));
  } else {
    const int u = blockIdx.y, f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.f_len[u]) return;
    r = (size_t)u * p.f_stride + f;
  }
  const double *row = p.in + r * p.row;
  double *out = p.out + r * p.dims;
  for (int b = 0; b < p.dims; ++b) {                                                // :231-236
    const int k = __ldg(p.idx + b);
    const double y0 = 20 * log10(row[k]);
    const double dy = (k + 1 < p.bins) ? 20 * log10(row[k + 1]) - y0 : 0.0;        // interp1Q: delta of the last node is 0
    out[b] = y0 + dy * __ldg(p.frac + b);
  }
}

// 128 threads (launch_frames); 16 CTAs per SM is full occupancy, at most 32 registers
WB_KERNEL(128, 16) decode_ap_kernel(CodecParams p) {
  const DecodeAt at = decode_at(p);
  if (at.f >= p.f_len[at.u]) return;
  const int n_ap = p.dims;
  const double *c = p.in + at.row * n_ap;
  double *out = p.out + at.row * p.row;
  double mean = 0.0;
  for (int b = 0; b < n_ap; ++b) mean += c[b];                                      // CheckVUV :32-40
  mean /= n_ap;
  const bool unvoiced = mean > -0.5;
  for (int j = threadIdx.x; j < p.bins; j += blockDim.x) {
    if (unvoiced) { out[j] = 1.0 - kCodecSafeGuardMinimum; continue; }              // :21-26, :263-264
    const int k = __ldg(p.idx + j);   // coarse nodes: 0 -> -60 dB, 1..n_ap -> coded, n_ap + 1 -> -1e-12
    const double a = (k == 0) ? -60.0 : c[k - 1];
    const double b = (k + 1 == n_ap + 1) ? -kCodecSafeGuardMinimum : c[k];
    const double v = a + __ldg(p.frac + j) * (b - a);
    out[j] = pow(10.0, v / 20.0);                                                   // :53-54
  }
}

struct PcmParams { const unsigned char *pcm; int bytes; const int *x_len; int x_stride; double zero_line; double *x; };

// audioio.cpp:238-249: magnitude of the low bits, minus 2^(nbit-1) when the sign bit is set
WB_DEV double pcm_sample(const unsigned char *s, int bytes, double zero_line) {
  unsigned v = 0;
  for (int j = bytes - 1; j >= 0; --j) v = v * 256u + s[j];
  const unsigned sign = 1u << (8 * bytes - 1);
  const double mag = static_cast<double>(v & (sign - 1u));
  const double bias = (v & sign) ? zero_line : 0.0;
  return (mag - bias) / zero_line;
}

WB_KERNEL_PLAIN pcm_kernel(PcmParams p) {
  const int u = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.x_len[u]) return;
  p.x[(size_t)u * p.x_stride + i] = pcm_sample(p.pcm + ((size_t)u * p.x_stride + i) * p.bytes, p.bytes, p.zero_line);
}

// packed samples -> padded float64 rows: utterance u (blockIdx.y) is samples [x_off[u], x_off[u + 1]) of src
WB_KERNEL_PLAIN gather_kernel(const unsigned char *__restrict__ src, int bytes, double zero_line,
                              const long long *__restrict__ x_off, int x_stride, double *__restrict__ out) {
  const int u = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long at = x_off[u] + i;
  if (at >= x_off[u + 1]) return;
  double *o = out + (size_t)u * x_stride + i;
  if (bytes == 0) *o = reinterpret_cast<const double *>(src)[at];
  else *o = pcm_sample(src + (size_t)at * bytes, bytes, zero_line);
}

int gather_samples(Ctx *ctx, const void *x, int nbit, const long long *x_off, int m, int max_len, int x_stride,
                   double *out) {
  const double zero_line = nbit ? pow(2.0, nbit - 1) : 1.0;
  for (int u0 = 0; u0 < m; u0 += 65535) {
    const int n = imin(65535, m - u0);
    WB_LAUNCH_FLAT(gather_kernel, dim3((unsigned)((max_len + 255) / 256), (unsigned)n), 256, 0, ctx->stream,
                   (const unsigned char *)x, nbit / 8, zero_line, x_off + u0, x_stride, out + (size_t)u0 * x_stride);
  }
  return dev_check(ctx, "gather");
}

// ---------------------------------------------------------------------------------- host side
namespace {

double frequency_to_mel(double f) { return kCodecM0 * log(f / kCodecF0 + 1.0); }   // codec.cpp:60-62
double mel_to_frequency(double m) { return kCodecF0 * (exp(m / kCodecM0) - 1.0); } // :67-69

// interp1's node selection (histc, matlabfunctions.cpp:136-155): k = smallest c >= 1 with xi < x[c],
// clamped to nx - 1; returns the left node k - 1 and the fraction of :170.
void interp1_tables(const std::vector<double> &x, const std::vector<double> &xi, std::vector<int> *idx,
                    std::vector<double> *frac) {
  const int nx = (int)x.size();
  idx->resize(xi.size());
  frac->resize(xi.size());
  int k = 1;
  for (size_t i = 0; i < xi.size(); ++i) {     // xi ascending, like every caller in codec.cpp
    while (k < nx - 1 && !(xi[i] < x[k])) ++k;
    (*idx)[i] = k - 1;
    (*frac)[i] = (xi[i] - x[k - 1]) / (x[k] - x[k - 1]);
  }
}

int check_fft(Ctx *ctx, int fft_size, int *lg_half) {
  int lg = 0;
  while ((1 << lg) < fft_size) ++lg;
  if ((1 << lg) != fft_size || fft_size < 16 || fft_size > WB_TW_N) {
    ctx->last_error = "codec: fft_size must be a power of two in [16, 8192]";
    return WORLD_B200_EINVAL;
  }
  *lg_half = lg - 1;
  return 0;
}

typedef CodecTables Tables;

// one launch per <= 65535 utterances; p carries the device tables, f_len the device lengths, max_f their largest
void launch_frames(Ctx *ctx, int which, CodecParams p, const int *f_len, int n_utts, int max_f, size_t in_row,
                   size_t out_row, size_t smem) {
  p.tw = ctx->twiddle;
#ifndef WB_EMU
  if (which == 0) cudaFuncSetAttribute(code_sp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (which == 1) cudaFuncSetAttribute(decode_sp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  const double *in = p.in;
  double *out = p.out;
  for (int u0 = 0; u0 < n_utts; u0 += 65535) {
    const int n = imin(65535, n_utts - u0);
    p.f_len = f_len + u0;
    p.in = in + (size_t)u0 * p.f_stride * in_row;
    p.out = out + (size_t)u0 * p.f_stride * out_row;
    if (which == 0) WB_LAUNCH_COOP(code_sp_kernel<false>, dim3((unsigned)max_f, (unsigned)n), 128, smem, ctx->stream, p);
    if (which == 1) WB_LAUNCH_COOP(decode_sp_kernel, dim3((unsigned)max_f, (unsigned)n), 128, smem, ctx->stream, p);
    if (which == 2) WB_LAUNCH_FLAT(code_ap_kernel, dim3((unsigned)((max_f + 127) / 128), (unsigned)n), 128, 0, ctx->stream, p);
    if (which == 3) WB_LAUNCH_FLAT(decode_ap_kernel, dim3((unsigned)max_f, (unsigned)n), 128, 0, ctx->stream, p);
  }
}

// lengths + tables into one arena block, then launch_frames
int run_frames(Ctx *ctx, int which, CodecParams p, const Tables &t, const int *f0_lengths, int n_utts,
               size_t in_row, size_t out_row, size_t smem) {
  if (n_utts == 0) return 0;
  std::vector<int> lens(n_utts);
  int max_f = 0;
  for (int i = 0; i < n_utts; ++i) {
    lens[i] = f0_lengths ? f0_lengths[i] : p.f_stride;
    if (lens[i] < 0 || lens[i] > p.f_stride) { ctx->last_error = "codec: f0_length outside its padded row"; return WORLD_B200_EINVAL; }
    if (lens[i] > max_f) max_f = lens[i];
  }
  if (max_f == 0) return 0;
  ArenaPlan plan;
  const size_t o_len = plan.add((size_t)n_utts * 4), o_idx = plan.add(t.idx.size() * 4 + 4);
  const size_t o_frac = plan.add(t.frac.size() * 8 + 8), o_w = plan.add(t.weight.size() * 16 + 16);
  unsigned char *blk = arena_block(ctx, plan.total);
  if (!blk) return WORLD_B200_ENOMEM;
  int rc = dev_memcpy_h2d(ctx, blk + o_len, lens.data(), lens.size() * 4);
  if (!rc && !t.idx.empty()) rc = dev_memcpy_h2d(ctx, blk + o_idx, t.idx.data(), t.idx.size() * 4);
  if (!rc && !t.frac.empty()) rc = dev_memcpy_h2d(ctx, blk + o_frac, t.frac.data(), t.frac.size() * 8);
  if (!rc && !t.weight.empty()) rc = dev_memcpy_h2d(ctx, blk + o_w, t.weight.data(), t.weight.size() * 16);
  if (rc) return rc;
  p.idx = (const int *)(blk + o_idx); p.frac = (const double *)(blk + o_frac);
  p.weight = (const double2 *)(blk + o_w);
  launch_frames(ctx, which, p, (const int *)(blk + o_len), n_utts, max_f, in_row, out_row, smem);
  return dev_check(ctx, "codec");
}

// the launch arguments of DecodeSpectralEnvelope (which 1) / DecodeAperiodicity (which 3) over tables t
CodecParams decode_params(int which, const Tables &t, int fft_size, int f_stride, const double *in, double *out) {
  CodecParams p;
  memset(&p, 0, sizeof(p));
  const int M = fft_size / 2;
  p.f_stride = f_stride; p.in = in; p.out = out; p.bins = M + 1; p.row = M + 1; p.dims = t.dims;
  if (which == 1) { p.max_dim = M; p.lg = t.lg_half; p.norm = t.norm; }
  return p;
}

size_t decode_smem(int which, int fft_size) {
  const int M = fft_size / 2;
  return which == 1 ? (size_t)(2 * M + M + 2) * 8 : 0;
}

}  // namespace

static int number_of_aperiodicities(int fs) {   // codec.cpp:216-219
  return static_cast<int>(dmin(kCodecUpperLimit, fs / 2.0 - kCodecFrequencyInterval) / kCodecFrequencyInterval);
}

// GetParametersForDecoding (codec.cpp:186-211) + the IDCT weights of DecodeSpectralEnvelope (:97-107)
int codec_decode_sp_tables(Ctx *ctx, int fs, int fft_size, int number_of_dimensions, CodecTables *t) {
  int lg = 0;
  int rc = check_fft(ctx, fft_size, &lg);
  if (rc) return rc;
  const int M = fft_size / 2;
  if (number_of_dimensions < 1 || number_of_dimensions > M) {
    ctx->last_error = "DecodeSpectralEnvelope: number_of_dimensions must be in [1, fft_size/2]";
    return WORLD_B200_EINVAL;
  }
  const double floor_mel = frequency_to_mel(kCodecFloorFrequency);
  const double ceil_mel = frequency_to_mel(dmin(fs / 2.0, kCodecCeilFrequency));
  t->weight.resize(number_of_dimensions);
  for (int i = 0; i < number_of_dimensions; ++i)
    t->weight[i] = make_double2(cos(i * kPi / fft_size) * sqrt((double)fft_size),
                                sin(i * kPi / fft_size) * sqrt((double)fft_size));
  t->weight[0].x /= sqrt(2.0);
  std::vector<double> mel_axis(M + 2), frequency_axis(M + 1);
  for (int i = 0; i < M; ++i) mel_axis[i + 1] = mel_to_frequency((ceil_mel - floor_mel) * i / M + floor_mel);
  mel_axis[0] = 0;
  mel_axis[M + 1] = fs / 2.0;
  for (int i = 0; i < M + 1; ++i) frequency_axis[i] = static_cast<double>(i) * fs / fft_size;
  interp1_tables(mel_axis, frequency_axis, &t->idx, &t->frac);
  t->dims = number_of_dimensions; t->lg_half = lg; t->norm = sqrt((double)M);
  return 0;
}

// interp1 over DecodeAperiodicity's coarse axis {0, 3k, ..., fs/2} (codec.cpp:244-251)
void codec_decode_ap_tables(int fs, int fft_size, CodecTables *t) {
  const int n_ap = number_of_aperiodicities(fs);
  const int bins = fft_size / 2 + 1;
  std::vector<double> frequency_axis(bins), coarse(n_ap + 2);
  for (int i = 0; i <= fft_size / 2; ++i) frequency_axis[i] = static_cast<double>(fs) / fft_size * i;
  for (int i = 0; i <= n_ap; ++i) coarse[i] = i * kCodecFrequencyInterval;
  coarse[n_ap + 1] = fs / 2.0;
  interp1_tables(coarse, frequency_axis, &t->idx, &t->frac);
  t->dims = n_ap;
}

void codec_decode_launch(Ctx *ctx, bool spectral_envelope, const CodecTables &t, const CodecDeviceTables &d,
                         int fft_size, const int *f_len, int n_utts, int f_stride, int max_f, const double *in,
                         double *out, const int *list, int out_row) {
  if (n_utts == 0 || max_f == 0) return;
  const int which = spectral_envelope ? 1 : 3;
  CodecParams p = decode_params(which, t, fft_size, f_stride, in, out);
  p.idx = d.idx; p.frac = d.frac; p.weight = d.weight;
  if (out_row) p.row = out_row;
  p.list = list;   // a list (at most one pass of utterances, < 65536) is one launch over the whole rows
  launch_frames(ctx, which, p, f_len, n_utts, max_f, t.dims, p.row, decode_smem(which, fft_size));
}

void codec_decode_packed_launch(Ctx *ctx, bool spectral_envelope, const CodecTables &t, const CodecDeviceTables &d,
                                int fft_size, const int *f_len, const long long *f_off, const int *list,
                                int list_n, const long long *cum, long long frames, const double *in, double *out,
                                int out_row) {
  if (list_n == 0 || frames == 0) return;
  const int which = spectral_envelope ? 1 : 3;
  CodecParams p = decode_params(which, t, fft_size, 0, in, out);
  p.idx = d.idx; p.frac = d.frac; p.weight = d.weight;
  p.row = out_row; p.list = list; p.f_off = f_off; p.cum = cum; p.list_n = list_n;
  p.tw = ctx->twiddle; p.f_len = f_len;   // every frame of the grid is within its utterance's f_len
  const size_t smem = decode_smem(which, fft_size);
#ifndef WB_EMU
  if (which == 1) cudaFuncSetAttribute(decode_sp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  if (which == 1) WB_LAUNCH_COOP(decode_sp_kernel, dim3((unsigned)frames), 128, smem, ctx->stream, p);
  else WB_LAUNCH_FLAT(decode_ap_kernel, dim3((unsigned)frames), 128, 0, ctx->stream, p);
}

// GetParametersForCoding (codec.cpp:161-181) + the DCT weights of DCTForCodec (:73-89)
int codec_sp_tables(Ctx *ctx, int fs, int fft_size, int number_of_dimensions, CodecTables *t) {
  int lg = 0;
  int rc = check_fft(ctx, fft_size, &lg);
  if (rc) return rc;
  const int M = fft_size / 2;
  if (number_of_dimensions < 1 || number_of_dimensions > M / 2 + 1) {
    ctx->last_error = "CodeSpectralEnvelope: number_of_dimensions must be in [1, fft_size/4 + 1]";
    return WORLD_B200_EINVAL;
  }
  const double floor_mel = frequency_to_mel(kCodecFloorFrequency);
  const double ceil_mel = frequency_to_mel(dmin(fs / 2.0, kCodecCeilFrequency));
  std::vector<double> mel_axis(M), frequency_axis(M + 1);
  t->weight.resize(number_of_dimensions);
  for (int i = 0; i < M; ++i) mel_axis[i] = (ceil_mel - floor_mel) * i / M + floor_mel;
  for (int i = 0; i < number_of_dimensions; ++i)
    t->weight[i] = make_double2(2.0 * cos(i * kPi / fft_size) / sqrt((double)fft_size),
                                2.0 * sin(i * kPi / fft_size) / sqrt((double)fft_size));
  t->weight[0].x /= sqrt(2.0);
  for (int i = 0; i <= M; ++i) frequency_axis[i] = frequency_to_mel(static_cast<double>(i) * fs / fft_size);
  interp1_tables(frequency_axis, mel_axis, &t->idx, &t->frac);
  t->dims = number_of_dimensions; t->lg_half = lg; t->norm = sqrt((double)M);
  return 0;
}

// interp1Q(0, fs / fft_size, ..., 3000 (i + 1)) of CodeAperiodicity (codec.cpp:228-238, matlabfunctions.cpp:214-235)
int codec_ap_tables(Ctx *ctx, int fs, int fft_size, CodecTables *t) {
  const int n_ap = number_of_aperiodicities(fs);
  t->dims = n_ap > 0 ? n_ap : 0;
  t->idx.resize(t->dims); t->frac.resize(t->dims);
  const double dx = static_cast<double>(fs) / fft_size;
  for (int i = 0; i < t->dims; ++i) {
    const double xi = kCodecFrequencyInterval * (i + 1.0);
    const int base = static_cast<int>((xi - 0) / dx);
    t->idx[i] = base;
    t->frac[i] = (xi - 0) / dx - base;
    if (base < 0 || base > fft_size / 2) { ctx->last_error = "CodeAperiodicity: band centre beyond fs/2"; return WORLD_B200_EINVAL; }
  }
  return 0;
}

// The packed codec calls (which: 0 CodeSpectralEnvelope, 1 DecodeSpectralEnvelope, 2 CodeAperiodicity,
// 3 DecodeAperiodicity): utterance u is frames [f_offsets[u], f_offsets[u + 1]) of its full rows ([F][row_stride], 0:
// the largest fft_sizes[u] / 2 + 1) and of its coded rows ([F][dims]).  Every check runs first, with the padded call's
// rules at each utterance's size; then the utterances are grouped by fft_size, in order of first appearance, and each
// group's frames are one launch in which entry j of the group's list owns frames [cum[j], cum[j + 1]) of the grid.
static int codec_packed(WorldB200 *h, int which, const double *in, int n, const long long *f_offsets, int row_stride,
                        const int *fft_sizes, int fs, int dims, double *out) {
  static const char *const names[4] = {"code_spectral_envelope_packed", "decode_spectral_envelope_packed",
                                       "code_aperiodicity_packed", "decode_aperiodicity_packed"};
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  auto fail = [&](const std::string &what, int u = -1) {
    ctx->last_error = std::string(names[which]) + ": " + what;
    if (u >= 0) ctx->last_error += " (utterance " + std::to_string(u) + ")";
    return WORLD_B200_EINVAL;
  };
  const bool sp = which < 2, code = which == 0 || which == 2;
  if (n < 0 || fs <= 0) return fail("n_utts must be >= 0 and fs > 0");
  if (!fft_sizes) return fail("fft_sizes must be given");
  const int n_ap = number_of_aperiodicities(fs);
  // the coded rows of the aperiodicity are empty below 12 kHz: CodeAperiodicity writes nothing, and its decode reads
  // nothing (a NULL array is allowed there)
  const double *coded = code ? out : in;
  std::vector<int> f_len;
  const std::string bad = packed_lengths("f_offsets", "frames", n, f_offsets, 0, &f_len);
  if (!bad.empty()) return fail(bad);
  // empty arrays may be NULL: a batch without frames reads and writes nothing
  if (n > 0 && f_offsets[n] > 0 && (!(code ? in : out) || (!coded && (sp || n_ap > 0))))
    return fail("the input and output rows must be given");
  std::vector<int> sizes, table(n);   // the distinct sizes, and each utterance's entry
  std::vector<Tables> tables;
  int row = row_stride;
  for (int u = 0; u < n; ++u) {
    const int f = fft_sizes[u];
    if (!sp && f < 2) return fail("fft_size must be at least 2", u);
    if (!row_stride) row = imax(row, f / 2 + 1);
    table[u] = (int)(std::find(sizes.begin(), sizes.end(), f) - sizes.begin());
    if (table[u] < (int)sizes.size()) continue;
    sizes.push_back(f);
    tables.emplace_back();
    const int rc = which == 0   ? codec_sp_tables(ctx, fs, f, dims, &tables.back())
                   : which == 1 ? codec_decode_sp_tables(ctx, fs, f, dims, &tables.back())
                   : which == 2 ? codec_ap_tables(ctx, fs, f, &tables.back())
                                : (codec_decode_ap_tables(fs, f, &tables.back()), 0);
    if (rc) {   // the table builder's message names its codec function already
      ctx->last_error += " (utterance " + std::to_string(u) + ")";
      return rc;
    }
  }
  for (int u = 0; u < n; ++u)
    if (row < fft_sizes[u] / 2 + 1) return fail("row_stride is smaller than fft_size / 2 + 1", u);
  if (which == 2 && n_ap <= 0) return 0;   // nothing to write below 12 kHz, like the reference's empty loops
  int rc = 0;
  for (size_t s = 0; s < sizes.size() && !rc; ++s) {
    const Tables &t = tables[s];
    const int fft_size = sizes[s], M = fft_size / 2;
    std::vector<int> list;
    std::vector<long long> cum(1, 0);
    for (int u = 0; u < n; ++u)
      if (table[u] == (int)s && f_len[u] > 0) { list.push_back(u); cum.push_back(cum.back() + f_len[u]); }
    const long long frames = cum.back();
    if (frames == 0) continue;
    const int m = (int)list.size();
    ArenaPlan plan;
    const size_t o_off = plan.add((size_t)(n + 1) * 8), o_cum = plan.add((size_t)(m + 1) * 8);
    const size_t o_len = plan.add((size_t)n * 4), o_list = plan.add((size_t)m * 4);
    const size_t o_idx = plan.add(t.idx.size() * 4 + 4), o_frac = plan.add(t.frac.size() * 8 + 8);
    const size_t o_w = plan.add(t.weight.size() * 16 + 16);
    unsigned char *blk = arena_block(ctx, plan.total);
    if (!blk) return WORLD_B200_ENOMEM;
    rc = dev_memcpy_h2d(ctx, blk + o_off, f_offsets, (size_t)(n + 1) * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_cum, cum.data(), cum.size() * 8);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_len, f_len.data(), (size_t)n * 4);
    if (!rc) rc = dev_memcpy_h2d(ctx, blk + o_list, list.data(), (size_t)m * 4);
    if (!rc && !t.idx.empty()) rc = dev_memcpy_h2d(ctx, blk + o_idx, t.idx.data(), t.idx.size() * 4);
    if (!rc && !t.frac.empty()) rc = dev_memcpy_h2d(ctx, blk + o_frac, t.frac.data(), t.frac.size() * 8);
    if (!rc && !t.weight.empty()) rc = dev_memcpy_h2d(ctx, blk + o_w, t.weight.data(), t.weight.size() * 16);
    if (rc) return rc;
    const long long *f_off = (const long long *)(blk + o_off), *cum_dev = (const long long *)(blk + o_cum);
    const int *f_len_dev = (const int *)(blk + o_len), *list_dev = (const int *)(blk + o_list);
    const CodecDeviceTables d{(const int *)(blk + o_idx), (const double *)(blk + o_frac),
                              (const double2 *)(blk + o_w)};
    if (!code) {
      codec_decode_packed_launch(ctx, sp, t, d, fft_size, f_len_dev, f_off, list_dev, m, cum_dev, frames,
                                 coded ? coded : out, out, row);
    } else {
      CodecParams p;
      memset(&p, 0, sizeof(p));
      p.in = in; p.out = out; p.bins = M + 1; p.row = row; p.dims = t.dims;
      p.idx = d.idx; p.frac = d.frac; p.weight = d.weight; p.tw = ctx->twiddle;
      p.f_len = f_len_dev; p.f_off = f_off; p.list = list_dev; p.cum = cum_dev; p.list_n = m;
      if (sp) {
        p.max_dim = M; p.lg = t.lg_half; p.norm = t.norm;
        const size_t smem = (size_t)(((M + 3) & ~1) + M + 2) * 8;
#ifndef WB_EMU
        cudaFuncSetAttribute(code_sp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
        WB_LAUNCH_COOP(code_sp_kernel<true>, dim3((unsigned)frames), 128, smem, ctx->stream, p);
      } else {
        WB_LAUNCH_FLAT(code_ap_kernel, dim3((unsigned)((frames + 127) / 128)), 128, 0, ctx->stream, p);
      }
    }
    rc = dev_check(ctx, "codec");
  }
  return rc;
}

}  // namespace wb

using namespace wb;

extern "C" {

int GetNumberOfAperiodicities(int fs) { return number_of_aperiodicities(fs); }

int world_b200_code_spectral_envelope_packed(WorldB200 *h, const double *spectrogram, int n_utts,
                                             const long long *f_offsets, int row_stride, const int *fft_sizes, int fs,
                                             int number_of_dimensions, double *coded_spectral_envelope) {
  return codec_packed(h, 0, spectrogram, n_utts, f_offsets, row_stride, fft_sizes, fs, number_of_dimensions,
                      coded_spectral_envelope);
}

int world_b200_decode_spectral_envelope_packed(WorldB200 *h, const double *coded_spectral_envelope, int n_utts,
                                               const long long *f_offsets, int row_stride, const int *fft_sizes,
                                               int fs, int number_of_dimensions, double *spectrogram) {
  return codec_packed(h, 1, coded_spectral_envelope, n_utts, f_offsets, row_stride, fft_sizes, fs,
                      number_of_dimensions, spectrogram);
}

int world_b200_code_aperiodicity_packed(WorldB200 *h, const double *aperiodicity, int n_utts,
                                        const long long *f_offsets, int row_stride, const int *fft_sizes, int fs,
                                        double *coded_aperiodicity) {
  return codec_packed(h, 2, aperiodicity, n_utts, f_offsets, row_stride, fft_sizes, fs, 0, coded_aperiodicity);
}

int world_b200_decode_aperiodicity_packed(WorldB200 *h, const double *coded_aperiodicity, int n_utts,
                                          const long long *f_offsets, int row_stride, const int *fft_sizes, int fs,
                                          double *aperiodicity) {
  return codec_packed(h, 3, coded_aperiodicity, n_utts, f_offsets, row_stride, fft_sizes, fs, 0, aperiodicity);
}

int world_b200_code_spectral_envelope_batch(WorldB200 *h, const double *spectrogram, int n_utts,
                                            const int *f0_lengths, int f0_stride, int fs, int fft_size,
                                            int number_of_dimensions, double *coded) {
  if (!h || !spectrogram || !coded || n_utts < 0 || fs <= 0 || f0_stride <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  Tables t;
  int rc = codec_sp_tables(ctx, fs, fft_size, number_of_dimensions, &t);
  if (rc) return rc;
  const int M = fft_size / 2, lg = t.lg_half;
  CodecParams p;
  memset(&p, 0, sizeof(p));
  p.f_stride = f0_stride; p.in = spectrogram; p.out = coded; p.bins = M + 1; p.row = M + 1;
  p.dims = number_of_dimensions; p.max_dim = M; p.lg = lg; p.norm = sqrt((double)M);
  const size_t smem = (size_t)(((M + 3) & ~1) + M + 2) * 8;
  return run_frames(ctx, 0, p, t, f0_lengths, n_utts, M + 1, number_of_dimensions, smem);
}

int world_b200_decode_spectral_envelope_batch(WorldB200 *h, const double *coded, int n_utts,
                                              const int *f0_lengths, int f0_stride, int fs, int fft_size,
                                              int number_of_dimensions, double *spectrogram) {
  if (!h || !spectrogram || !coded || n_utts < 0 || fs <= 0 || f0_stride <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  Tables t;
  const int rc = codec_decode_sp_tables(ctx, fs, fft_size, number_of_dimensions, &t);
  if (rc) return rc;
  const CodecParams p = decode_params(1, t, fft_size, f0_stride, coded, spectrogram);
  return run_frames(ctx, 1, p, t, f0_lengths, n_utts, number_of_dimensions, fft_size / 2 + 1, decode_smem(1, fft_size));
}

int world_b200_code_aperiodicity_batch(WorldB200 *h, const double *aperiodicity, int n_utts,
                                       const int *f0_lengths, int f0_stride, int fs, int fft_size, double *coded) {
  if (!h || !aperiodicity || n_utts < 0 || fs <= 0 || f0_stride <= 0 || fft_size < 2) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  const int n_ap = GetNumberOfAperiodicities(fs);
  if (n_ap <= 0) return 0;          // nothing to write below 12 kHz, like the reference's empty loops
  if (!coded) return WORLD_B200_EINVAL;
  Tables t;
  int rc = codec_ap_tables(ctx, fs, fft_size, &t);
  if (rc) return rc;
  CodecParams p;
  memset(&p, 0, sizeof(p));
  p.f_stride = f0_stride; p.in = aperiodicity; p.out = coded; p.bins = fft_size / 2 + 1; p.row = p.bins; p.dims = n_ap;
  return run_frames(ctx, 2, p, t, f0_lengths, n_utts, fft_size / 2 + 1, n_ap, 0);
}

int world_b200_decode_aperiodicity_batch(WorldB200 *h, const double *coded, int n_utts, const int *f0_lengths,
                                         int f0_stride, int fs, int fft_size, double *aperiodicity) {
  if (!h || !aperiodicity || n_utts < 0 || fs <= 0 || f0_stride <= 0 || fft_size < 2) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  const int n_ap = GetNumberOfAperiodicities(fs);
  if (n_ap < 0 || (n_ap > 0 && !coded)) return WORLD_B200_EINVAL;
  Tables t;
  codec_decode_ap_tables(fs, fft_size, &t);
  const CodecParams p = decode_params(3, t, fft_size, f0_stride, coded ? coded : aperiodicity, aperiodicity);
  return run_frames(ctx, 3, p, t, f0_lengths, n_utts, n_ap, fft_size / 2 + 1, decode_smem(3, fft_size));
}

int world_b200_wav_parse(const unsigned char *b, unsigned long long size, int *fs, int *nbit, int *n_samples,
                         unsigned long long *data_offset) {
  // RIFF <size> WAVE fmt <16> <format 1> <channels 1> <fs> <byte rate> <block align> <bits> ... data <bytes>
  if (!b || !fs || !nbit || !n_samples || !data_offset || size < 44) return WORLD_B200_EINVAL;
  if (memcmp(b, "RIFF", 4) || memcmp(b + 8, "WAVE", 4) || memcmp(b + 12, "fmt ", 4)) return WORLD_B200_EINVAL;
  if (!(b[16] == 16 && b[17] == 0 && b[18] == 0 && b[19] == 0)) return WORLD_B200_EINVAL;  // fmt chunk of 16 bytes
  if (!(b[20] == 1 && b[21] == 0)) return WORLD_B200_EINVAL;                                 // PCM
  if (!(b[22] == 1 && b[23] == 0)) return WORLD_B200_EINVAL;                                 // mono
  *fs = (int)(b[24] | (b[25] << 8) | (b[26] << 16) | ((unsigned)b[27] << 24));
  *nbit = b[34];
  if (*nbit != 8 && *nbit != 16 && *nbit != 24 && *nbit != 32) return WORLD_B200_EINVAL;
  unsigned long long pos = 36;   // first byte after the fmt chunk; scan for the "data" tag like the reference
  while (pos + 8 <= size && memcmp(b + pos, "data", 4)) ++pos;
  if (pos + 8 > size) return WORLD_B200_EINVAL;
  unsigned long long bytes = b[pos + 4] | (b[pos + 5] << 8) | (b[pos + 6] << 16) | ((unsigned long long)b[pos + 7] << 24);
  *data_offset = pos + 8;
  if (bytes > size - *data_offset) bytes = size - *data_offset;   // truncated file: what is there
  *n_samples = (int)(bytes / (unsigned)(*nbit / 8));
  return 0;
}

int world_b200_pcm_to_double_batch(WorldB200 *h, const void *pcm, int nbit, int n_utts, int x_stride,
                                   const int *x_lengths, double *x) {
  if (!h || !pcm || !x || n_utts < 0 || x_stride <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  if (nbit != 8 && nbit != 16 && nbit != 24 && nbit != 32) { ctx->last_error = "pcm: nbit must be 8, 16, 24 or 32"; return WORLD_B200_EINVAL; }
  if (n_utts == 0) return 0;
  std::vector<int> lens(n_utts);
  int mx = 0;
  for (int i = 0; i < n_utts; ++i) {
    lens[i] = x_lengths ? x_lengths[i] : x_stride;
    if (lens[i] < 0 || lens[i] > x_stride) { ctx->last_error = "pcm: x_length outside its padded row"; return WORLD_B200_EINVAL; }
    if (lens[i] > mx) mx = lens[i];
  }
  if (mx == 0) return 0;
  ArenaPlan plan;
  const size_t o_len = plan.add((size_t)n_utts * 4);
  unsigned char *blk = arena_block(ctx, plan.total);
  if (!blk) return WORLD_B200_ENOMEM;
  int rc = dev_memcpy_h2d(ctx, blk + o_len, lens.data(), lens.size() * 4);
  if (rc) return rc;
  for (int u0 = 0; u0 < n_utts; u0 += 65535) {
    const int n = imin(65535, n_utts - u0);
    PcmParams p;
    p.bytes = nbit / 8;
    p.pcm = (const unsigned char *)pcm + (size_t)u0 * x_stride * p.bytes;
    p.x_len = (const int *)(blk + o_len) + u0; p.x_stride = x_stride;
    p.zero_line = pow(2.0, nbit - 1);
    p.x = x + (size_t)u0 * x_stride;
    WB_LAUNCH_FLAT(pcm_kernel, dim3((unsigned)((mx + 255) / 256), (unsigned)n), 256, 0, ctx->stream, p);
  }
  return dev_check(ctx, "pcm_to_double");
}

}  // extern "C"
