/* world_b200.h -- batched C ABI of the GPU-native (H100, sm_90a) WORLD analysis engine.
 *
 * The reference (mmorise/World) has no plugin registry; its boundary is the public C API of
 * the src/world headers (SURVEY.md 8b).  That API is kept source-compatible in include/world/
 * (single utterance, host pointers).  This header is the thin extern "C" layer underneath it:
 * the same stages, N utterances per call, plain pointers and sizes, no C++/torch types.
 *
 * Conventions
 *   - Batches are padded row-major arrays:  x[n_utts][x_stride] (doubles in [-1,1]),
 *     time_axis / f0 [n_utts][f0_stride], spectrogram / aperiodicity
 *     [n_utts][f0_stride][fft_size/2+1].  Per-utterance valid lengths are HOST int arrays
 *     (x_lengths[n_utts], f0_lengths[n_utts]); NULL means "every row is full"
 *     (x_stride samples / f0_stride frames).  Padding is never read; padded frames are never
 *     written.
 *   - The *_batch functions take DEVICE pointers for the big arrays and enqueue their work on
 *     the context's stream (world_b200_set_stream); they do not synchronise.  One exception:
 *     world_b200_synthesis_batch, world_b200_synthesis_coded_batch and world_b200_synthesis_coded_batch_pcm16 read
 *     their pulse counts back once per chunk of utterances, which
 *     synchronises the context's stream (all work queued on it before the call included) before
 *     the chunk's remaining kernels are enqueued.  The *_host
 *     functions take host pointers, stage through device memory and return when the results are
 *     in the caller's buffers.
 *   - Every function returns 0 on success or a WORLD_B200_E* code; world_b200_last_error()
 *     describes the failure.  (The reference returns void and has undefined behaviour on bad
 *     input; the legacy wrappers in include/world/ keep `void` and print the message.)
 *   - Frame counts follow the reference exactly: world_b200_frames() ==
 *     GetSamplesForDIO()/GetSamplesForHarvest() (dio.cpp:639-641, harvest.cpp:1219-1221).
 */
#ifndef WORLD_B200_H_
#define WORLD_B200_H_

#include "world/dio.h"
#include "world/harvest.h"
#include "world/cheaptrick.h"
#include "world/d4c.h"
#include "world/stonemask.h"
#include "world/synthesis.h"
#include "world/codec.h"

#ifdef __cplusplus
extern "C" {
#endif

#define WORLD_B200_OK 0
#define WORLD_B200_ECUDA 1     /* a CUDA runtime call or kernel failed                        */
#define WORLD_B200_ENOMEM 2    /* device scratch could not be allocated                       */
#define WORLD_B200_EINVAL 3    /* argument outside what the on-chip kernels support           */
#define WORLD_B200_EDOMAIN 4   /* a frame hit a case that is undefined in the reference
                                  (e.g. f0 below the floor implied by fft_size), or an
                                  utterance needs more than the 2^31 randn() draws the library
                                  reproduces; see message                                      */

typedef struct WorldB200 WorldB200;

/* Creates a context on CUDA device `device` (tables, scratch arena, status word).  Fails with
 * WORLD_B200_ECUDA when no usable device exists: there is no CPU fallback. */
int world_b200_create(int device, WorldB200 **ctx);
void world_b200_destroy(WorldB200 *ctx);
/* cuda_stream is a cudaStream_t; NULL selects the default stream. */
int world_b200_set_stream(WorldB200 *ctx, void *cuda_stream);
/* Upper bound (bytes) of internal scratch one stage call may hold; batches are processed in
 * utterance chunks that fit it.  Default: a third of the memory free at creation, clamped to
 * [4, 64] GiB. */
int world_b200_set_scratch_budget(WorldB200 *ctx, unsigned long long bytes);
/* Synchronises and releases the device memory the context keeps between calls (scratch arena, the randn()
 * stream table and the staging buffers of the *_host pipelines); the next call allocates again. */
int world_b200_trim(WorldB200 *ctx);
int world_b200_synchronize(WorldB200 *ctx);
const char *world_b200_last_error(const WorldB200 *ctx);
/* Number of kernels this context has launched so far (bench.py reports it). */
unsigned long long world_b200_launch_count(const WorldB200 *ctx);

/* Per-kernel device timing (CUDA events on the context's stream around every launch).
 * profile(ctx, 1) starts collecting; profile_report() synchronises, writes a JSON object
 * {"<kernel>": {"launches": n, "ms": total}, ...} into buf and clears the collection. */
int world_b200_profile(WorldB200 *ctx, int enable);
int world_b200_profile_report(WorldB200 *ctx, char *buf, unsigned long long cap);

/* Measured FP64 FMA peak of the device in TFLOP/s (8 independent DFMA chains per thread, CUDA
 * events): the roofline the analysis path is bound by (no FP64 figure exists in MEASURED_PEAKS). */
int world_b200_fp64_peak(WorldB200 *ctx, double *tflops);

/* Measured FP64 tensor-core peak of the device in TFLOP/s: the same harness with 8 independent
 * mma.m16n8k4.f64 chains per warp (Harvest's band-pass filter bank runs on this pipe). */
int world_b200_fp64_tensor_peak(WorldB200 *ctx, double *tflops);

/* Test hook: forward real FFT of n = 2^k doubles (4 <= n <= 8192) with the library's shared-memory
 * FFT; out_dev receives n/2+1 interleaved complex values (n + 2 doubles).  DEVICE pointers. */
int world_b200_rfft_test(WorldB200 *ctx, const double *x_dev, int n, double *out_dev);
/* same, through the self-sorting padded FFT the frame kernels use since round 2 */
int world_b200_sfft_test(WorldB200 *ctx, const double *x_dev, int n, double *out_dev);

/* Test hook: first n_draws values of the reference's randn() stream (matlabfunctions.cpp:237-264)
 * as raw 32-bit sums (value = sum / 2^28 - 6) into a DEVICE buffer of n_draws uint32. */
int world_b200_randn_stream(WorldB200 *ctx, unsigned n_draws, unsigned *out_dev);
/* Test hook: draws [first, first + n) of the same stream, in the same form, into a DEVICE buffer of n
 * uint32.  The library reproduces the stream up to draw 2^31 of each utterance (first + n <= 2^31, else
 * EINVAL); a CheapTrick, D4C or Synthesis call whose utterance would draw more reports WORLD_B200_EDOMAIN
 * at world_b200_synchronize() rather than reuse the stream. */
int world_b200_randn_window(WorldB200 *ctx, unsigned long long first, unsigned n, unsigned *out_dev);

/* int(1000.0 * x_length / fs / frame_period) + 1 */
int world_b200_frames(int fs, int x_length, double frame_period);

/* ---- batched stages, device pointers -------------------------------------------------- */
/* Dio() over a batch (dio.h:38).  Writes time_axis and f0 rows of world_b200_frames() entries. */
int world_b200_dio_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                         const int *x_lengths, int fs, const DioOption *option,
                         double *time_axis, double *f0, int f0_stride);
/* The same with one option per utterance: dio_options is a HOST array of n_utts.  f0_floor, f0_ceil,
 * channels_in_octave and allowed_range may differ between utterances; frame_period and speed must be the same for all
 * (they fix the decimation, the low-cut filter and the frame grid; else EINVAL).  Each row equals what
 * world_b200_dio_batch gives that utterance with its own option.  A band list the on-chip kernels cannot serve is
 * EINVAL, and world_b200_last_error() names the first such utterance. */
int world_b200_dio_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                 const int *x_lengths, int fs, const DioOption *dio_options,
                                 double *time_axis, double *f0, int f0_stride);
/* Harvest() over a batch (harvest.h:35). */
int world_b200_harvest_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                             const int *x_lengths, int fs, const HarvestOption *option,
                             double *time_axis, double *f0, int f0_stride);
/* The same with one option per utterance: harvest_options is a HOST array of n_utts.  f0_floor / f0_ceil may differ
 * between utterances (a speaker's or singer's own range); frame_period must be the same for all (else EINVAL).  Each
 * row equals what world_b200_harvest_batch gives that utterance with its own option.  A range the on-chip kernels
 * cannot serve is EINVAL, and world_b200_last_error() names the first such utterance. */
int world_b200_harvest_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                     const int *x_lengths, int fs, const HarvestOption *harvest_options,
                                     double *time_axis, double *f0, int f0_stride);
/* StoneMask() over a batch (stonemask.h:27). refined_f0 may alias f0. */
int world_b200_stonemask_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                               const int *x_lengths, int fs, const double *time_axis,
                               const double *f0, const int *f0_lengths, int f0_stride,
                               double *refined_f0);
/* CheapTrick() over a batch (cheaptrick.h:38); option->fft_size selects the row width. */
int world_b200_cheaptrick_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                const int *x_lengths, int fs, const double *time_axis,
                                const double *f0, const int *f0_lengths, int f0_stride,
                                const CheapTrickOption *option, double *spectrogram);
/* D4C() over a batch (d4c.h:35); fft_size is CheapTrick's. */
int world_b200_d4c_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                         const int *x_lengths, int fs, const double *time_axis,
                         const double *f0, const int *f0_lengths, int f0_stride, int fft_size,
                         const D4COption *option, double *aperiodicity);

/* Synthesis() over a batch (synthesis.h:30) -- SURVEY.md 8 row f1.  f0 [n][f0_stride], spectrogram /
 * aperiodicity [n][f0_stride][fft_size/2+1], y [n][y_stride] (all DEVICE); f0_lengths / y_lengths are
 * host arrays (NULL = full rows).  frame_period in ms. */
int world_b200_synthesis_batch(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                               int f0_stride, const double *spectrogram, const double *aperiodicity,
                               int fft_size, double frame_period, int fs, const int *y_lengths,
                               int y_stride, double *y);

/* Synthesis() from coded rows: DecodeSpectralEnvelope() (codec.h:86) + DecodeAperiodicity() (codec.h:53) + Synthesis()
 * (synthesis.h:30) over a batch, without full-row arrays.  f0 [n][f0_stride], coded_spectral_envelope
 * [n][f0_stride][number_of_dimensions], coded_aperiodicity [n][f0_stride][GetNumberOfAperiodicities(fs)],
 * y [n][y_stride], all DEVICE; f0_lengths / y_lengths HOST or NULL (full rows).  frame_period in ms.
 *   - Output: every row equals, bit for bit, what world_b200_decode_spectral_envelope_batch +
 *     world_b200_decode_aperiodicity_batch + world_b200_synthesis_batch give for the same utterance (the same kernels
 *     run on the same values).  The rows are decoded chunk by chunk into the call's scratch, so the decoded rows of
 *     one chunk of utterances (16 * (fft_size/2+1) bytes per frame) are held at a time, never those of the batch.
 *   - Validation, before any work is queued (WORLD_B200_EINVAL): fft_size a power of two in [16, 4096];
 *     number_of_dimensions in [1, fft_size/2]; f0 and y lengths >= 2 and within their rows; coded_aperiodicity
 *     non-NULL whenever GetNumberOfAperiodicities(fs) > 0.
 *   - Below 12 kHz there are no aperiodicity bands: coded_aperiodicity may be NULL and is not read, and the
 *     aperiodicity decodes as world_b200_decode_aperiodicity_batch decodes zero bands (the reference's CheckVUV mean
 *     is 0/0, which takes the voiced branch, over the nodes {0 Hz: -60 dB, fs/2: -1e-12 dB}).
 *   - Stream behaviour is world_b200_synthesis_batch's, with its one exception: one read-back of the pulse counts per
 *     chunk of utterances, which synchronises the context's stream. */
int world_b200_synthesis_coded_batch(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                     int f0_stride, const double *coded_spectral_envelope,
                                     int number_of_dimensions, const double *coded_aperiodicity,
                                     int fft_size, double frame_period, int fs, const int *y_lengths,
                                     int y_stride, double *y);

/* world_b200_synthesis_coded_batch with 16-bit PCM out: the same arguments, checks and stream behaviour, but y is
 * [n][y_stride] int16 (DEVICE).  The overlap-add kernel stores wavwrite's quantisation (tools/audioio.cpp) of each
 * sample it sums, so the float64 waveform never reaches device memory (2 bytes per sample instead of 8):
 *     v = (int)(sample * 32767)   (truncation toward zero),   v = clamp(v, -32768, 32767).
 * Where |sample * 32767| < 2^31 every value equals the library's own wavwrite() of what
 * world_b200_synthesis_coded_batch writes for that sample, bit for bit.  Beyond that range the reference's int cast
 * is undefined behaviour; here such a sample saturates by its sign (-32768 or 32767), and NaN gives 0.  Padded
 * samples (beyond an utterance's y_length) are not written. */
int world_b200_synthesis_coded_batch_pcm16(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                           int f0_stride, const double *coded_spectral_envelope,
                                           int number_of_dimensions, const double *coded_aperiodicity,
                                           int fft_size, double frame_period, int fs, const int *y_lengths,
                                           int y_stride, short *y);

/* Synthesis from coded rows for HOST arrays, the counterpart of world_b200_analyze_coded_host: f0 [n][f0_stride],
 * coded_spectral_envelope [n][f0_stride][number_of_dimensions], coded_aperiodicity
 * [n][f0_stride][GetNumberOfAperiodicities(fs)] (may be NULL below 12 kHz), f0_lengths / y_lengths (or NULL) and y,
 * all HOST.  y is [n][y_stride] float64 for nbit 0 or int16 for nbit 16 (any other nbit is WORLD_B200_EINVAL).
 *   - Output: equal bit for bit to world_b200_synthesis_coded_batch (nbit 0) or
 *     world_b200_synthesis_coded_batch_pcm16 (nbit 16) for the same utterance.  Whole rows are written back: samples
 *     beyond an utterance's y_length read as 0.
 *   - Validation is that of world_b200_synthesis_coded_batch plus nbit, all before any work is queued; after an error
 *     y is unchanged.
 *   - Upload, synthesis and download are pipelined over utterance chunks on three streams (uploads, the context's
 *     stream, downloads); the call returns when the results are in y.  Pinned host buffers (cudaHostAlloc /
 *     cudaHostRegister) let the copies run under the kernels; pageable ones give the same results, with the copies
 *     serialised against the host. */
int world_b200_synthesis_coded_host(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                    int f0_stride, const double *coded_spectral_envelope, int number_of_dimensions,
                                    const double *coded_aperiodicity, int fft_size, double frame_period, int fs,
                                    const int *y_lengths, int y_stride, int nbit, void *y);

/* ---- voice modification: F0 scaling and formant shift (the reference demo's ParameterModification,
 * test/test.cpp:221-258), one factor per utterance --------------------------------------------------------------
 * For utterance u with shift = f0_scale[u], ratio = spectral_ratio[u] and bins = fft_size/2 + 1, every frame
 * i < f0_length is changed as the reference changes it:
 *     f0[i] *= shift                                   (unvoiced frames stay 0)
 *     sp[i][j] = exp(interp1(x, log(sp[i]), xi)[j])     x[m] = ratio * m / fft_size * fs, xi[m] = (double)m / fft_size * fs
 *     ratio < 1: sp[i][j] = sp[i][c - 1] for j >= c = (int)(fft_size / 2.0 * ratio)
 * (interp1 extrapolates with its last segment; ratio 1.0 still takes the log / exp round trip.)  Aperiodicity is not
 * changed, and nothing is analysed again: scale after all analysis, as the reference does.
 *   - f0 [n_utts][f0_stride] and spectrogram [n_utts][f0_stride][fft_size/2+1] are DEVICE rows, changed in place;
 *     f0_lengths is HOST or NULL (full rows); f0_scale and spectral_ratio are HOST arrays of n_utts.  Either may be
 *     NULL, which skips that half; f0 or spectrogram may then be NULL too.  Padding frames are never written.
 *   - The segment and weight of each bin are planned on the host once per distinct ratio (the reference's expressions
 *     and its histc), and the kernel rounds y[k-1] + s * (y[k] - y[k-1]) step by step, without FMA.  So f0 equals the
 *     reference bit for bit, and an envelope differs from it only through the device's log / exp (within 1e-12
 *     relative of the host's libm).
 *   - Validation, before any work is queued (WORLD_B200_EINVAL, world_b200_last_error() naming the first bad
 *     utterance): f0_lengths within [0, f0_stride]; a factor that is not finite or not > 0; with spectral_ratio,
 *     fft_size a power of two in [16, 4096], fs > 0, and no ratio with c == 0 (the reference would read sp[-1]).
 *   - Like the other *_batch stages the call does not synchronise. */
int world_b200_modify_batch(WorldB200 *ctx, double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                            double *spectrogram, int fft_size, int fs, const double *f0_scale,
                            const double *spectral_ratio);
/* world_b200_synthesis_coded_batch with the modification applied inside: the arguments of that call plus f0_scale and
 * spectral_ratio (HOST arrays of n_utts, NULL = none) and nbit (0: y is float64, 16: y is int16 quantised as
 * world_b200_synthesis_coded_batch_pcm16 quantises; anything else is EINVAL).  The caller's f0 and coded rows are not
 * changed: each chunk of utterances synthesises from a scaled copy of its f0 rows (held in the call's scratch, so
 * the time base, the pulse count and a relaid pass all see the scaled contour) and stretches its decoded envelope
 * block right after the decode.
 *   - Output: equal bit for bit to world_b200_decode_spectral_envelope_batch -> world_b200_modify_batch ->
 *     world_b200_decode_aperiodicity_batch -> world_b200_synthesis_batch for the same utterance (nbit 0), or to the
 *     pcm16 rule applied to that waveform (nbit 16).  With both arrays NULL it is world_b200_synthesis_coded_batch /
 *     _pcm16, on exactly their path.
 *   - Validation is that of world_b200_synthesis_coded_batch and of world_b200_modify_batch, all before any work is
 *     queued.  Stream behaviour as world_b200_synthesis_coded_batch. */
int world_b200_synthesis_coded_batch_modified(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                              int f0_stride, const double *coded_spectral_envelope,
                                              int number_of_dimensions, const double *coded_aperiodicity,
                                              int fft_size, double frame_period, int fs, const int *y_lengths,
                                              int y_stride, const double *f0_scale, const double *spectral_ratio,
                                              int nbit, void *y);
/* The same for HOST arrays through the pipeline of world_b200_synthesis_coded_host (which slices f0_scale and
 * spectral_ratio with the utterance chunks): equal bit for bit to world_b200_synthesis_coded_batch_modified. */
int world_b200_synthesis_coded_host_modified(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                             int f0_stride, const double *coded_spectral_envelope,
                                             int number_of_dimensions, const double *coded_aperiodicity,
                                             int fft_size, double frame_period, int fs, const int *y_lengths,
                                             int y_stride, const double *f0_scale, const double *spectral_ratio,
                                             int nbit, void *y);

/* ---- Synthesis with one fft_size per utterance: the way back from world_b200_cheaptrick_batch_options /
 * world_b200_d4c_batch_options (full rows) and world_b200_analyze_coded_*_spectral_options (coded rows).
 * fft_sizes is a HOST array of n_utts: utterance u is synthesised at fft_sizes[u], a power of two in [16, 4096] -- the
 * size that sets its lowest_f0 = fs / fft_size + 1, its DC remover, its response length and its decode tables, as the
 * reference demo's Synthesis call with CheapTrick's fft_size.  The sizes may come in any order.
 *   - Output: every row equals, bit for bit, the one-size call of the same family (world_b200_synthesis_batch,
 *     world_b200_synthesis_coded_batch_modified, world_b200_synthesis_coded_host_modified, world_b200_modify_batch) on
 *     that utterance alone at fft_sizes[u].  A call whose sizes are all equal is that call.
 *   - Validation, before any work is queued (WORLD_B200_EINVAL, world_b200_last_error() naming the first bad
 *     utterance): fft_sizes non-NULL and each a power of two in [16, 4096]; full rows: row_stride >= fft_sizes[u]/2 + 1
 *     for every u; coded rows: number_of_dimensions in [1, fft_sizes[u]/2] for every u; then the checks of the one-size
 *     call.  Stream behaviour as that call's. */
/* spectrogram / aperiodicity [n][f0_stride][row_stride] (DEVICE), of which utterance u reads fft_sizes[u]/2 + 1 values
 * per frame: the layout the *_batch_options stages write.  Otherwise world_b200_synthesis_batch. */
int world_b200_synthesis_batch_options(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                       int f0_stride, const double *spectrogram, const double *aperiodicity,
                                       int row_stride, const int *fft_sizes, double frame_period, int fs,
                                       const int *y_lengths, int y_stride, double *y);
/* Coded rows as world_b200_synthesis_coded_batch_modified (f0_scale / spectral_ratio may be NULL; nbit 0: float64 y,
 * 16: int16 y), each utterance decoded and synthesised at its own size.  The pulse responses of a pass are computed in
 * one launch per distinct size; the decoded rows of a pass are laid out at the largest size's bins. */
int world_b200_synthesis_coded_batch_options(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                             int f0_stride, const double *coded_spectral_envelope,
                                             int number_of_dimensions, const double *coded_aperiodicity,
                                             const int *fft_sizes, double frame_period, int fs, const int *y_lengths,
                                             int y_stride, const double *f0_scale, const double *spectral_ratio,
                                             int nbit, void *y);
/* The same for HOST arrays through the pipeline of world_b200_synthesis_coded_host. */
int world_b200_synthesis_coded_host_options(WorldB200 *ctx, const double *f0, const int *f0_lengths, int n_utts,
                                            int f0_stride, const double *coded_spectral_envelope,
                                            int number_of_dimensions, const double *coded_aperiodicity,
                                            const int *fft_sizes, double frame_period, int fs, const int *y_lengths,
                                            int y_stride, const double *f0_scale, const double *spectral_ratio,
                                            int nbit, void *y);
/* world_b200_modify_batch on spectrogram rows [n][f0_stride][row_stride] (DEVICE): utterance u's envelope is the first
 * fft_sizes[u]/2 + 1 values of each row, stretched with its own size (the stretch tables are planned once per distinct
 * (ratio, fft_size)).  fft_sizes and row_stride are read only with spectral_ratio. */
int world_b200_modify_batch_options(WorldB200 *ctx, double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                                    double *spectrogram, int row_stride, const int *fft_sizes, int fs,
                                    const double *f0_scale, const double *spectral_ratio);

/* ---- codec over a batch (codec.h:20-92) -- SURVEY.md 8 row f2; all DEVICE pointers ------ */
/* aperiodicity [n][f0_stride][fft_size/2+1] -> coded [n][f0_stride][GetNumberOfAperiodicities(fs)]. */
int world_b200_code_aperiodicity_batch(WorldB200 *ctx, const double *aperiodicity, int n_utts,
                                       const int *f0_lengths, int f0_stride, int fs, int fft_size,
                                       double *coded_aperiodicity);
int world_b200_decode_aperiodicity_batch(WorldB200 *ctx, const double *coded_aperiodicity, int n_utts,
                                         const int *f0_lengths, int f0_stride, int fs, int fft_size,
                                         double *aperiodicity);
/* spectrogram [n][f0_stride][fft_size/2+1] -> coded [n][f0_stride][number_of_dimensions]. */
int world_b200_code_spectral_envelope_batch(WorldB200 *ctx, const double *spectrogram, int n_utts,
                                            const int *f0_lengths, int f0_stride, int fs, int fft_size,
                                            int number_of_dimensions, double *coded_spectral_envelope);
int world_b200_decode_spectral_envelope_batch(WorldB200 *ctx, const double *coded_spectral_envelope,
                                              int n_utts, const int *f0_lengths, int f0_stride, int fs,
                                              int fft_size, int number_of_dimensions, double *spectrogram);
/* CheapTrick() + CodeSpectralEnvelope() (cheaptrick.h:38, codec.h:62-64) and D4C() + CodeAperiodicity()
 * (d4c.h:35, codec.h:33-34) in ONE kernel per frame: the coded row is computed in the frame kernel's shared memory
 * and the fft_size/2+1 bin rows are never written.  Arguments as in world_b200_cheaptrick_batch /
 * world_b200_d4c_batch; coded_spectral_envelope [n][f0_stride][number_of_dimensions], coded_aperiodicity
 * [n][f0_stride][GetNumberOfAperiodicities(fs)] (DEVICE).  Same values as the two-step path up to the rounding of
 * the exp/log (10^x/log10) pair that cancels. */
int world_b200_cheaptrick_coded_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                      const int *x_lengths, int fs, const double *time_axis,
                                      const double *f0, const int *f0_lengths, int f0_stride,
                                      const CheapTrickOption *option, int number_of_dimensions,
                                      double *coded_spectral_envelope);
int world_b200_d4c_coded_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                               const int *x_lengths, int fs, const double *time_axis,
                               const double *f0, const int *f0_lengths, int f0_stride, int fft_size,
                               const D4COption *option, double *coded_aperiodicity);

/* CheapTrick and D4C with one option per utterance, so each speaker of a batch gets the FFT size of its own F0 floor
 * (CheapTrick analyses a frame at or below 3 fs / (fft_size - 3) as if it were at 500 Hz).  Derive the sizes as the
 * reference does: options[u].f0_floor = floor[u]; options[u].fft_size = GetFFTSizeForCheapTrick(fs, &options[u]);
 * f0_floor itself is not read.  options, fft_sizes: HOST arrays of n_utts; every other array as in the one-option
 * calls.  Full rows: spectrogram / aperiodicity [n][f0_stride][row_stride] (DEVICE), row_stride >= the largest
 * fft_sizes[u] / 2 + 1; utterance u writes the first fft_size_u / 2 + 1 values of each of its rows and leaves the rest
 * of the row untouched.  Coded rows keep the one-option layout (number_of_dimensions, resp.
 * GetNumberOfAperiodicities(fs), values per frame whatever the size), so a mixed batch lands in one array.
 * Every row equals, bit for bit, what the one-option call gives that utterance with its own option; with equal
 * options the call equals the one-option call.  CheapTrick runs one launch sequence per distinct option, D4C one for
 * the batch.  Checked before any work is queued (EINVAL, world_b200_last_error() naming the first bad utterance,
 * outputs untouched): CheapTrick fft_size a power of two in [16, 8192], D4C fft_size >= 4, q1 / threshold finite,
 * row_stride, and number_of_dimensions in [1, fft_size / 4 + 1] for every utterance's size. */
int world_b200_cheaptrick_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                        const int *x_lengths, int fs, const double *time_axis,
                                        const double *f0, const int *f0_lengths, int f0_stride,
                                        const CheapTrickOption *options, int row_stride, double *spectrogram);
int world_b200_d4c_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                 const int *x_lengths, int fs, const double *time_axis,
                                 const double *f0, const int *f0_lengths, int f0_stride, const int *fft_sizes,
                                 const D4COption *options, int row_stride, double *aperiodicity);
int world_b200_cheaptrick_coded_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                              const int *x_lengths, int fs, const double *time_axis,
                                              const double *f0, const int *f0_lengths, int f0_stride,
                                              const CheapTrickOption *options, int number_of_dimensions,
                                              double *coded_spectral_envelope);
int world_b200_d4c_coded_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                       const int *x_lengths, int fs, const double *time_axis,
                                       const double *f0, const int *f0_lengths, int f0_stride,
                                       const int *fft_sizes, const D4COption *options,
                                       double *coded_aperiodicity);

/* ---- ingest (tools/audioio.cpp:217-252) -- SURVEY.md 8 row f3 --------------------------- */
/* Host-only: locates the sample data of a mono PCM RIFF/WAVE image held in memory, with the
 * acceptance rules of the reference's wavread (16-byte fmt chunk, format 1, one channel). */
int world_b200_wav_parse(const unsigned char *bytes, unsigned long long size, int *fs, int *nbit,
                         int *n_samples, unsigned long long *data_offset);
/* Little-endian signed PCM of nbit in {8, 16, 24, 32}, rows [n][x_stride] samples (DEVICE), to the
 * doubles wavread produces: sample / 2^(nbit-1), exact.  x_lengths NULL = full rows. */
int world_b200_pcm_to_double_batch(WorldB200 *ctx, const void *pcm, int nbit, int n_utts, int x_stride,
                                   const int *x_lengths, double *x);

/* ---- whole analysis chain, host pointers ---------------------------------------------- */
#define WORLD_B200_F0_DIO_STONEMASK 0
#define WORLD_B200_F0_HARVEST 1

typedef struct {
  int f0_method;                 /* WORLD_B200_F0_*                                  */
  DioOption dio;                 /* used when f0_method == DIO_STONEMASK             */
  HarvestOption harvest;         /* used when f0_method == HARVEST                   */
  CheapTrickOption cheaptrick;
  D4COption d4c;
} WorldB200AnalysisOption;

void world_b200_default_analysis_option(int fs, int f0_method, WorldB200AnalysisOption *option);

/* The whole chain on DEVICE arrays (layouts as above; x_lengths HOST or NULL): {Dio+StoneMask | Harvest} ->
 * CheapTrick -> D4C.  The batch is cut into utterance slices that alternate between two internal streams, so the
 * latency-bound per-utterance kernels of one slice run under the FP64-bound kernels of the other.  The work is
 * ordered after what is already on the context's stream, and that stream waits for it: like the *_batch stages the
 * call does not synchronise the host.  spectrogram / aperiodicity may be NULL to stop after the F0 stage / after
 * CheapTrick.  Each internal stream may use half the scratch budget. */
int world_b200_analyze_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                             const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                             double *time_axis, double *f0, int f0_stride, double *spectrogram,
                             double *aperiodicity);
/* The same chain with one Harvest option per utterance (harvest_options: HOST array of n_utts, see
 * world_b200_harvest_batch_options; the slices split it with the utterances).  option->f0_method must be
 * WORLD_B200_F0_HARVEST and every harvest_options[u].frame_period must equal option->harvest.frame_period (else
 * EINVAL); option->harvest's floor and ceiling are not used.  The *_options variants below follow the same rules. */
int world_b200_analyze_batch_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                     const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                     const HarvestOption *harvest_options, double *time_axis, double *f0,
                                     int f0_stride, double *spectrogram, double *aperiodicity);
/* ... with one DIO option per utterance (dio_options: HOST array of n_utts, see world_b200_dio_batch_options).
 * option->f0_method must be WORLD_B200_F0_DIO_STONEMASK, and every dio_options[u].frame_period and .speed must equal
 * option->dio's (else EINVAL); option->dio's floor, ceiling, channels_in_octave and allowed_range are not used.  The
 * *_dio_options variants below follow the same rules.  Options of the other F0 method are EINVAL. */
int world_b200_analyze_batch_dio_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                         const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                         const DioOption *dio_options, double *time_axis, double *f0,
                                         int f0_stride, double *spectrogram, double *aperiodicity);
/* ... with per-utterance spectral options, so each speaker's full rows come from the FFT size of its own F0 floor:
 * cheaptrick_options and d4c_options are HOST arrays of n_utts (either may be NULL: option->cheaptrick / option->d4c
 * for every utterance), harvest_options / dio_options as above (at most one, of the chain's F0 method, or both NULL).
 * CheapTrick runs at cheaptrick_options[u].fft_size and D4C at the same size.  spectrogram / aperiodicity are
 * [n_utts][f0_stride][row_stride] (DEVICE), one stride for both, as in world_b200_cheaptrick_batch_options /
 * world_b200_d4c_batch_options: row_stride >= every utterance's fft_size / 2 + 1 (0: the largest of them).  Utterance
 * u writes the first fft_size_u / 2 + 1 values of each of its frames; the rest of each row, and every frame past the
 * utterance's count, are left untouched.  Each row equals, bit for bit, what world_b200_analyze_batch gives that
 * utterance with its own options; with equal options and row_stride = fft_size / 2 + 1 the call equals
 * world_b200_analyze_batch.  Checked before any work is queued (EINVAL, world_b200_last_error() naming the first bad
 * utterance, outputs untouched): the rules of the stage calls with options, those of the *_options / *_dio_options
 * chains, and row_stride. */
int world_b200_analyze_batch_spectral_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                              const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                              const HarvestOption *harvest_options, const DioOption *dio_options,
                                              const CheapTrickOption *cheaptrick_options,
                                              const D4COption *d4c_options, double *time_axis, double *f0,
                                              int f0_stride, int row_stride, double *spectrogram,
                                              double *aperiodicity);

/* ---- multi-GPU: one context per GPU (one process or thread each), utterances sharded over ranks --------------
 * There is no exchange inside the analysis; the one collective reassembles the output arrays on every rank
 * (north_star; reference loops src/harvest.cpp:1223-1255, cheaptrick.cpp:200-229, d4c.cpp:342-403 are per utterance).
 * NCCL is bound at run time (dlopen of libnccl.so.2) -- single-GPU users never load it.  Rank 0 creates the id and
 * the CALLER hands its 128 bytes to the other ranks (MPI, torch.distributed, a socket, a file ...). */
int world_b200_comm_unique_id(unsigned char *id, int id_bytes /* >= 128 */);
int world_b200_comm_init(WorldB200 *ctx, int n_ranks, int rank, const unsigned char *id, int id_bytes);
int world_b200_comm_destroy(WorldB200 *ctx);
/* In-place all-gather: `full` is [n_ranks][rows_per_rank][row_elems] doubles (DEVICE) with this rank's block already
 * in place.  Ordered after the work on the context's stream; that stream waits for the result. */
int world_b200_allgather_rows(WorldB200 *ctx, double *full, unsigned long long row_elems,
                              unsigned long long rows_per_rank);
/* world_b200_analyze_batch on this rank's n_utts utterances (every rank passes the same n_utts, strides and options),
 * with the four outputs given as the FULL arrays of n_ranks * n_utts utterances: the rank computes into its own
 * block and each finished utterance slice is sent to all other ranks while the next slice is computed -- the
 * transfer hides under the compute.  Transport: the rank copies its rows into the peers' arrays, mapped through CUDA
 * IPC (copy engines over NVLink, no SM involved; the handles are exchanged once per set of arrays through the
 * communicator, which briefly synchronises the communication stream with the host), or, where the arrays cannot be
 * exported, grouped ncclBroadcasts on a high-priority stream (WB_NO_P2P=1 forces this).  Collective: every rank
 * must make the call.  On return the work is enqueued; after the context's stream (world_b200_synchronize) every
 * rank holds the complete arrays, bit-identical to a single-GPU run. */
int world_b200_analyze_batch_allgather(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                       const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                       double *time_axis_full, double *f0_full, int f0_stride,
                                       double *spectrogram_full, double *aperiodicity_full);
/* ... with one Harvest option per utterance of THIS rank's shard (harvest_options: HOST array of n_utts).  The ranges
 * may differ between ranks; n_utts, strides, fs and option must still be the same on every rank. */
int world_b200_analyze_batch_allgather_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                               const int *x_lengths, int fs,
                                               const WorldB200AnalysisOption *option,
                                               const HarvestOption *harvest_options, double *time_axis_full,
                                               double *f0_full, int f0_stride, double *spectrogram_full,
                                               double *aperiodicity_full);
/* ... with one DIO option per utterance of THIS rank's shard (dio_options: HOST array of n_utts). */
int world_b200_analyze_batch_allgather_dio_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                                   const int *x_lengths, int fs,
                                                   const WorldB200AnalysisOption *option,
                                                   const DioOption *dio_options, double *time_axis_full,
                                                   double *f0_full, int f0_stride, double *spectrogram_full,
                                                   double *aperiodicity_full);
/* ... with per-utterance spectral options of THIS rank's shard, as world_b200_analyze_batch_spectral_options: the
 * full arrays are [n_ranks * n_utts][f0_stride][row_stride].  The shards' largest fft_sizes may differ, so the rows
 * need one stride for all ranks: every rank passes the same n_utts, f0_stride and row_stride, with row_stride >= the
 * largest fft_size / 2 + 1 of ALL ranks (0 means this rank's largest, which is only safe when every rank's largest
 * size is the same).  Collective. */
int world_b200_analyze_batch_allgather_spectral_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                                        const int *x_lengths, int fs,
                                                        const WorldB200AnalysisOption *option,
                                                        const HarvestOption *harvest_options,
                                                        const DioOption *dio_options,
                                                        const CheapTrickOption *cheaptrick_options,
                                                        const D4COption *d4c_options, double *time_axis_full,
                                                        double *f0_full, int f0_stride, int row_stride,
                                                        double *spectrogram_full, double *aperiodicity_full);

/* {Dio+StoneMask | Harvest} -> CheapTrick -> D4C for n_utts host waveforms; outputs are host
 * arrays laid out as described above.  Input upload, compute and result download are pipelined
 * over utterance chunks.  Any output pointer may be NULL to skip its download.  Whole padded rows
 * are downloaded: frames beyond an utterance's own count come back as zeros. */
int world_b200_analyze_host(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                            const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                            double *time_axis, double *f0, int f0_stride, double *spectrogram,
                            double *aperiodicity);
/* ... with one Harvest option per utterance (HOST array of n_utts; the chunks split it). */
int world_b200_analyze_host_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                    const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                    const HarvestOption *harvest_options, double *time_axis, double *f0,
                                    int f0_stride, double *spectrogram, double *aperiodicity);
/* ... with one DIO option per utterance (HOST array of n_utts; the chunks split it). */
int world_b200_analyze_host_dio_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                        const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                        const DioOption *dio_options, double *time_axis, double *f0,
                                        int f0_stride, double *spectrogram, double *aperiodicity);
/* ... with per-utterance spectral options and F0 options as world_b200_analyze_batch_spectral_options, its rows
 * [n_utts][f0_stride][row_stride] in HOST arrays.  Whole padded rows are downloaded: the values past an utterance's
 * fft_size / 2 + 1, and the frames past its count, come back as zeros.  Every computed value equals the device call's. */
int world_b200_analyze_host_spectral_options(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                                             const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                             const HarvestOption *harvest_options, const DioOption *dio_options,
                                             const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                             double *time_axis, double *f0, int f0_stride, int row_stride,
                                             double *spectrogram, double *aperiodicity);

/* The same chain with the ingest and the codec fused in on the device: x holds samples of `nbit`
 * bits (0 = doubles as above; 8/16/24/32 = little-endian PCM as in a WAV data chunk), and the
 * results that cross PCIe are the coded rows -- coded_spectral_envelope [n][f0_stride]
 * [number_of_dimensions], coded_aperiodicity [n][f0_stride][GetNumberOfAperiodicities(fs)] -- about
 * 8.4 times (16 kHz, 60 dimensions) fewer device-to-host bytes than the full rows. */
int world_b200_analyze_coded_host(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                  const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                  int number_of_dimensions, double *time_axis, double *f0, int f0_stride,
                                  double *coded_spectral_envelope, double *coded_aperiodicity);
/* ... with one option per utterance of the chain's F0 method (HOST array of n_utts; the chunks split it): Harvest
 * options as for world_b200_analyze_host_options, DIO options as for world_b200_analyze_host_dio_options. */
int world_b200_analyze_coded_host_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                          const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                          const HarvestOption *harvest_options, int number_of_dimensions,
                                          double *time_axis, double *f0, int f0_stride,
                                          double *coded_spectral_envelope, double *coded_aperiodicity);
int world_b200_analyze_coded_host_dio_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                              const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                              const DioOption *dio_options, int number_of_dimensions,
                                              double *time_axis, double *f0, int f0_stride,
                                              double *coded_spectral_envelope, double *coded_aperiodicity);

/* The coded chain on DEVICE arrays: world_b200_analyze_batch with the input and output formats of
 * world_b200_analyze_coded_host.  x (DEVICE) holds rows of x_stride samples of `nbit` bits (0 = doubles; 8/16/24/32 =
 * little-endian PCM, converted exactly as world_b200_pcm_to_double_batch does; a row is x_stride * nbit/8 bytes);
 * x_lengths is HOST or NULL.  time_axis / f0 are [n_utts][f0_stride], coded_spectral_envelope is
 * [n_utts][f0_stride][number_of_dimensions] and coded_aperiodicity [n_utts][f0_stride][GetNumberOfAperiodicities(fs)],
 * all DEVICE; frames beyond an utterance's own count are not written.  Only the coded rows reach device memory (the
 * frame kernels code them), so the outputs are number_of_dimensions and GetNumberOfAperiodicities(fs) doubles per frame
 * instead of 2 * (fft_size/2 + 1).  coded_spectral_envelope NULL skips CheapTrick, coded_aperiodicity NULL skips D4C;
 * below 12 kHz there are no aperiodicity bands and D4C is skipped (coded_aperiodicity may be NULL).  Every row equals
 * world_b200_analyze_coded_host's for the same utterance and options, bit for bit.  Bad nbit, number_of_dimensions
 * outside [1, fft_size/4 + 1], per-utterance options that break the rules of world_b200_analyze_batch_options /
 * _dio_options, or lengths outside their rows are EINVAL before any work is queued.  Stream behaviour and the two
 * internal streams as for world_b200_analyze_batch; with PCM input each internal stream also holds one float64 buffer
 * of its largest slice, taken from its half of the scratch budget. */
int world_b200_analyze_coded_batch(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                   const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                   int number_of_dimensions, double *time_axis, double *f0, int f0_stride,
                                   double *coded_spectral_envelope, double *coded_aperiodicity);
/* ... with one Harvest option per utterance (HOST array of n_utts), as world_b200_analyze_batch_options. */
int world_b200_analyze_coded_batch_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                           const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                           const HarvestOption *harvest_options, int number_of_dimensions,
                                           double *time_axis, double *f0, int f0_stride,
                                           double *coded_spectral_envelope, double *coded_aperiodicity);
/* ... with one DIO option per utterance (HOST array of n_utts), as world_b200_analyze_batch_dio_options. */
int world_b200_analyze_coded_batch_dio_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                               const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                               const DioOption *dio_options, int number_of_dimensions,
                                               double *time_axis, double *f0, int f0_stride,
                                               double *coded_spectral_envelope, double *coded_aperiodicity);
/* ... with per-utterance spectral options as well: cheaptrick_options and d4c_options are HOST arrays of n_utts (either
 * may be NULL: option->cheaptrick / option->d4c for every utterance), harvest_options / dio_options as above (at most
 * one, of the chain's F0 method, or both NULL).  CheapTrick runs at cheaptrick_options[u].fft_size and D4C at the same
 * size, as in world_b200_cheaptrick_coded_batch_options / world_b200_d4c_coded_batch_options, whose rules are checked
 * for every utterance before any work is queued (number_of_dimensions against every utterance's size).  Each row equals
 * what world_b200_analyze_coded_batch gives that utterance with its own options, bit for bit. */
int world_b200_analyze_coded_batch_spectral_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                                    const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                                    const HarvestOption *harvest_options, const DioOption *dio_options,
                                                    const CheapTrickOption *cheaptrick_options,
                                                    const D4COption *d4c_options, int number_of_dimensions,
                                                    double *time_axis, double *f0, int f0_stride,
                                                    double *coded_spectral_envelope, double *coded_aperiodicity);
/* The same for HOST arrays, on world_b200_analyze_coded_host's pipeline: each row equals
 * world_b200_analyze_coded_batch_spectral_options's for the same utterance and options, bit for bit. */
int world_b200_analyze_coded_host_spectral_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                                   const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                                   const HarvestOption *harvest_options, const DioOption *dio_options,
                                                   const CheapTrickOption *cheaptrick_options,
                                                   const D4COption *d4c_options, int number_of_dimensions,
                                                   double *time_axis, double *f0, int f0_stride,
                                                   double *coded_spectral_envelope, double *coded_aperiodicity);
/* world_b200_analyze_coded_batch on this rank's n_utts utterances with the outputs given as the FULL arrays of
 * n_ranks * n_utts utterances, gathered on every rank as world_b200_analyze_batch_allgather gathers the full rows:
 * the exchanged rows are the coded ones (f0_stride * number_of_dimensions and f0_stride * GetNumberOfAperiodicities(fs)
 * doubles per utterance), and an array that is NULL or has no bands is not exchanged.  Collective. */
int world_b200_analyze_coded_batch_allgather(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                             const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                             int number_of_dimensions, double *time_axis_full, double *f0_full,
                                             int f0_stride, double *coded_spectral_envelope_full,
                                             double *coded_aperiodicity_full);
/* ... with one Harvest option per utterance of THIS rank's shard (HOST array of n_utts). */
int world_b200_analyze_coded_batch_allgather_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                                     const int *x_lengths, int fs,
                                                     const WorldB200AnalysisOption *option,
                                                     const HarvestOption *harvest_options, int number_of_dimensions,
                                                     double *time_axis_full, double *f0_full, int f0_stride,
                                                     double *coded_spectral_envelope_full,
                                                     double *coded_aperiodicity_full);
/* ... with one DIO option per utterance of THIS rank's shard (HOST array of n_utts). */
int world_b200_analyze_coded_batch_allgather_dio_options(WorldB200 *ctx, const void *x, int nbit, int n_utts,
                                                         int x_stride, const int *x_lengths, int fs,
                                                         const WorldB200AnalysisOption *option,
                                                         const DioOption *dio_options, int number_of_dimensions,
                                                         double *time_axis_full, double *f0_full, int f0_stride,
                                                         double *coded_spectral_envelope_full,
                                                         double *coded_aperiodicity_full);
/* ... with per-utterance spectral options of THIS rank's shard, as world_b200_analyze_coded_batch_spectral_options.
 * Coded rows do not depend on the size, so the shards' sizes may differ freely; every rank passes the same n_utts,
 * f0_stride and number_of_dimensions, which must fit every utterance's size on every rank.  Collective. */
int world_b200_analyze_coded_batch_allgather_spectral_options(
    WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths, int fs,
    const WorldB200AnalysisOption *option, const HarvestOption *harvest_options, const DioOption *dio_options,
    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options, int number_of_dimensions,
    double *time_axis_full, double *f0_full, int f0_stride, double *coded_spectral_envelope_full,
    double *coded_aperiodicity_full);

/* ---- packed batches: utterances back to back, no padding ----------------------------------------------------------
 * x_offsets: a HOST array of n_utts + 1 sample offsets, x_offsets[0] == 0: utterance u is samples
 * [x_offsets[u], x_offsets[u + 1]) of x (with PCM input, byte offset = sample offset * nbit / 8).  Each utterance is
 * 1 .. INT_MAX samples long.  Its frames follow on from the previous utterance's:
 *   f_offsets[0] = 0, f_offsets[u + 1] = f_offsets[u] + world_b200_frames(fs, len_u, frame_period),
 * frame_period being the chain's F0 method's, and F = f_offsets[n_utts] frames in all.  time_axis and f0 are [F];
 * full rows are [F][row_stride] (row_stride >= every utterance's fft_size / 2 + 1; 0: the largest); coded rows
 * [F][number_of_dimensions] and [F][GetNumberOfAperiodicities(fs)]. */
/* f_offsets (HOST, n_utts + 1) of a packed batch, to size its outputs before the call.  EINVAL for bad offsets. */
int world_b200_packed_frames(int fs, int n_utts, const long long *x_offsets, double frame_period,
                             long long *f_offsets);
/* world_b200_analyze_batch_spectral_options on a packed batch (DEVICE arrays).  Every utterance's time axis, f0 and
 * rows equal, bit for bit, what the padded call gives it with the same options.  Nothing is written outside frames
 * [0, F), nor past an utterance's fft_size / 2 + 1 in a full row.  f_offsets (HOST, n_utts + 1, may be NULL) receives
 * the frame offsets.  Checked before any work is queued: the padded call's rules and the offset rules (EINVAL,
 * world_b200_last_error() naming the first bad utterance, outputs untouched).  n_utts == 0 writes f_offsets[0] = 0. */
int world_b200_analyze_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                              const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                              const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                              const D4COption *d4c_options, double *time_axis, double *f0, int row_stride,
                              double *spectrogram, double *aperiodicity, long long *f_offsets);
/* world_b200_analyze_coded_batch_spectral_options on a packed batch of nbit 0/8/16/24/32 samples (DEVICE arrays),
 * as world_b200_analyze_packed. */
int world_b200_analyze_coded_packed(WorldB200 *ctx, const void *x, int nbit, int n_utts, const long long *x_offsets,
                                    int fs, const WorldB200AnalysisOption *option,
                                    const HarvestOption *harvest_options, const DioOption *dio_options,
                                    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                    int number_of_dimensions, double *time_axis, double *f0,
                                    double *coded_spectral_envelope, double *coded_aperiodicity,
                                    long long *f_offsets);
/* The same two chains for HOST arrays.  Each chunk of utterances goes up as one contiguous copy of its samples and
 * comes back as one contiguous copy per output array; no padding crosses PCIe.  Exactly F frames are written, and full
 * rows read 0 past an utterance's fft_size / 2 + 1.  time_axis and f0 may be NULL (not downloaded). */
int world_b200_analyze_host_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                                   const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                                   const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                                   const D4COption *d4c_options, double *time_axis, double *f0, int row_stride,
                                   double *spectrogram, double *aperiodicity, long long *f_offsets);
int world_b200_analyze_coded_host_packed(WorldB200 *ctx, const void *x, int nbit, int n_utts,
                                         const long long *x_offsets, int fs, const WorldB200AnalysisOption *option,
                                         const HarvestOption *harvest_options, const DioOption *dio_options,
                                         const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                         int number_of_dimensions, double *time_axis, double *f0,
                                         double *coded_spectral_envelope, double *coded_aperiodicity,
                                         long long *f_offsets);

/* The way back on packed rows.  f_offsets and y_offsets are HOST arrays of n_utts + 1 offsets starting at 0:
 * utterance u is frames [f_offsets[u], f_offsets[u + 1]) of f0 / the rows and samples [y_offsets[u], y_offsets[u + 1])
 * of y.  f_offsets may be the array world_b200_analyze_*packed returns, and y_offsets = x_offsets gives the output the
 * input's layout.  fft_sizes (HOST, n_utts) is required, as in the _options calls.  Every address is 64-bit: F,
 * F * row_stride and Y may exceed 2^31.
 * Equality: utterance u's samples equal, bit for bit, what the padded call of the same family gives it with the same
 * fft_sizes, f0_lengths[u] = f_offsets[u + 1] - f_offsets[u] and y_lengths[u] = y_offsets[u + 1] - y_offsets[u]:
 * world_b200_synthesis_batch_options, world_b200_synthesis_coded_batch_options, world_b200_modify_batch_options.
 * Checked before any work is queued: the padded call's rules, offsets starting at 0, and for synthesis 2 .. INT_MAX
 * frames and samples per utterance (modification: 0 .. INT_MAX frames); EINVAL, world_b200_last_error() naming the
 * first bad utterance, outputs untouched.  n_utts == 0 returns 0. */
/* Synthesis on packed rows (DEVICE arrays): f0 [F]; spectrogram / aperiodicity [F][row_stride] (0: the largest
 * fft_sizes[u] / 2 + 1); y [Y] float64, Y = y_offsets[n_utts].  Writes samples [0, Y) of y and nothing else. */
int world_b200_synthesis_packed(WorldB200 *ctx, const double *f0, int n_utts, const long long *f_offsets,
                                const double *spectrogram, const double *aperiodicity, int row_stride,
                                const int *fft_sizes, double frame_period, int fs, const long long *y_offsets,
                                double *y);
/* Synthesis from coded rows [F][number_of_dimensions] and [F][GetNumberOfAperiodicities(fs)] (DEVICE arrays).
 * f0_scale / spectral_ratio (HOST, n_utts) may be NULL.  nbit 0: y is float64; nbit 16: int16, quantised as wavwrite
 * does.  Writes samples [0, Y) of y and nothing else. */
int world_b200_synthesis_coded_packed(WorldB200 *ctx, const double *f0, int n_utts, const long long *f_offsets,
                                      const double *coded_spectral_envelope, int number_of_dimensions,
                                      const double *coded_aperiodicity, const int *fft_sizes, double frame_period,
                                      int fs, const long long *y_offsets, const double *f0_scale,
                                      const double *spectral_ratio, int nbit, void *y);
/* The same for HOST arrays, pipelined: each chunk's frames go up as one copy per input array and its samples come back
 * as one copy.  Writes exactly Y samples; its output equals world_b200_synthesis_coded_packed's. */
int world_b200_synthesis_coded_host_packed(WorldB200 *ctx, const double *f0, int n_utts, const long long *f_offsets,
                                           const double *coded_spectral_envelope, int number_of_dimensions,
                                           const double *coded_aperiodicity, const int *fft_sizes,
                                           double frame_period, int fs, const long long *y_offsets,
                                           const double *f0_scale, const double *spectral_ratio, int nbit, void *y);
/* ParameterModification in place on packed rows (DEVICE arrays): f0 [F], spectrogram [F][row_stride] (0: the largest
 * fft_sizes[u] / 2 + 1; fft_sizes may be NULL when spectral_ratio is).  Writes nothing outside frames [0, F), nor past
 * an utterance's fft_size / 2 + 1 in a row. */
int world_b200_modify_packed(WorldB200 *ctx, double *f0, int n_utts, const long long *f_offsets, double *spectrogram,
                             int row_stride, const int *fft_sizes, int fs, const double *f0_scale,
                             const double *spectral_ratio);

/* ---- pitch and formant curves: one f0 factor and one spectral ratio per FRAME ---------------------------------------
 * Frame i of an utterance is modified exactly as ParameterModification (test.cpp:221-258) modifies a one-frame
 * spectrogram with shift = f0_curve[i] and ratio = spectral_ratio_curve[i] at the utterance's fft_size.  The curves are
 * DEVICE arrays laid out as f0: [n_utts][f0_stride] for world_b200_modify_curves, [F] at f_offsets for
 * world_b200_modify_curves_packed; either may be NULL, which skips that half.  Rows, lengths, sizes and row_stride are
 * those of world_b200_modify_batch_options / world_b200_modify_packed (fft_sizes may be NULL without a ratio curve).
 * Constant curves (curve[i] = factor[u] on every frame of utterance u) give world_b200_modify_batch_options /
 * world_b200_modify_packed's result with those factors, bit for bit.  Writes nothing outside the utterances' frames
 * (frames [0, F) packed), nor past an utterance's fft_size / 2 + 1 in a row.
 * Validation, before any modification is queued (WORLD_B200_EINVAL, world_b200_last_error() naming the curve, index,
 * utterance, frame and value; the rows are unchanged): the rules of the factor calls, and per frame an f0 factor that is
 * not finite and > 0, or a ratio that is not finite and > 0 or has (int)(fft_size / 2.0 * ratio) < 1.  The curves are
 * checked where they are, on the device, by one small kernel: these calls synchronise the stream once.  n_utts == 0
 * returns 0. */
int world_b200_modify_curves(WorldB200 *ctx, double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                             double *spectrogram, int row_stride, const int *fft_sizes, int fs, const double *f0_curve,
                             const double *spectral_ratio_curve);
int world_b200_modify_curves_packed(WorldB200 *ctx, double *f0, int n_utts, const long long *f_offsets,
                                    double *spectrogram, int row_stride, const int *fft_sizes, int fs,
                                    const double *f0_curve, const double *spectral_ratio_curve);

/* The stage calls on packed batches (DEVICE arrays), for callers who bring their own F0 or rows.  x_offsets and
 * f_offsets are HOST arrays of n_utts + 1 offsets, each starting at 0: utterance u is samples
 * [x_offsets[u], x_offsets[u + 1]) of x (1 .. INT_MAX of them) and frames [f_offsets[u], f_offsets[u + 1]) of time_axis,
 * f0 and every output (0 .. INT_MAX of them).  f_offsets is the caller's: world_b200_packed_frames or
 * world_b200_analyze_packed give one, but an F0 at another hop has its own frame counts.  Options and sizes are HOST
 * arrays of n_utts and are required (a batch of one option repeats it); d4c_options may be NULL (InitializeD4COption).
 * Full rows are [F][row_stride] (0: the largest fft_size / 2 + 1); coded rows [F][number_of_dimensions] and
 * [F][GetNumberOfAperiodicities(fs)].  Every address is 64-bit.  The kernels read x, time_axis and f0 where they are:
 * no padded copy is made.
 * Equality: utterance u's output equals, bit for bit, what the padded call of the same family gives it with the same
 * option and f0_lengths[u] = f_offsets[u + 1] - f_offsets[u]: world_b200_stonemask_batch,
 * world_b200_cheaptrick_batch_options, world_b200_cheaptrick_coded_batch_options, world_b200_d4c_batch_options,
 * world_b200_d4c_coded_batch_options, and the *_batch codec call at the utterance's fft_size.
 * Nothing is written outside frames [0, F), nor past an utterance's fft_size / 2 + 1 in a full row.  Checked before any
 * work is queued: the padded call's rules, offsets that start at 0 and never decrease, and a row_stride wide enough for
 * every utterance's size; EINVAL, world_b200_last_error() naming the first bad utterance, outputs untouched.  n_utts == 0
 * returns 0.  F0 alone on a packed batch is world_b200_analyze_packed / world_b200_analyze_coded_packed with NULL rows. */
/* StoneMask: refined_f0 [F] (may alias f0). */
int world_b200_stonemask_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                                const double *time_axis, const double *f0, const long long *f_offsets,
                                double *refined_f0);
int world_b200_cheaptrick_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                                 const double *time_axis, const double *f0, const long long *f_offsets,
                                 const CheapTrickOption *cheaptrick_options, int row_stride, double *spectrogram);
int world_b200_cheaptrick_coded_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                                       const double *time_axis, const double *f0, const long long *f_offsets,
                                       const CheapTrickOption *cheaptrick_options, int number_of_dimensions,
                                       double *coded_spectral_envelope);
/* D4C at each utterance's CheapTrick size fft_sizes[u]. */
int world_b200_d4c_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                          const double *time_axis, const double *f0, const long long *f_offsets, const int *fft_sizes,
                          const D4COption *d4c_options, int row_stride, double *aperiodicity);
/* Below 12 kHz there are no bands: nothing is written, and coded_aperiodicity may be NULL. */
int world_b200_d4c_coded_packed(WorldB200 *ctx, const double *x, int n_utts, const long long *x_offsets, int fs,
                                const double *time_axis, const double *f0, const long long *f_offsets,
                                const int *fft_sizes, const D4COption *d4c_options, double *coded_aperiodicity);
/* The codec between full rows [F][row_stride] and coded rows, each utterance at its own fft_sizes[u].  Below 12 kHz the
 * coded aperiodicity is empty (may be NULL): coding it writes nothing, decoding it writes the unvoiced rows. */
int world_b200_code_spectral_envelope_packed(WorldB200 *ctx, const double *spectrogram, int n_utts,
                                             const long long *f_offsets, int row_stride, const int *fft_sizes, int fs,
                                             int number_of_dimensions, double *coded_spectral_envelope);
int world_b200_decode_spectral_envelope_packed(WorldB200 *ctx, const double *coded_spectral_envelope, int n_utts,
                                               const long long *f_offsets, int row_stride, const int *fft_sizes,
                                               int fs, int number_of_dimensions, double *spectrogram);
int world_b200_code_aperiodicity_packed(WorldB200 *ctx, const double *aperiodicity, int n_utts,
                                        const long long *f_offsets, int row_stride, const int *fft_sizes, int fs,
                                        double *coded_aperiodicity);
int world_b200_decode_aperiodicity_packed(WorldB200 *ctx, const double *coded_aperiodicity, int n_utts,
                                          const long long *f_offsets, int row_stride, const int *fft_sizes, int fs,
                                          double *aperiodicity);

/* ---- voice transformation, PCM in and PCM out: the reference demo's loop (test/test.cpp: Harvest or DIO + StoneMask,
 * CheapTrick, D4C, ParameterModification, Synthesis) over a batch in one call, with one pitch, formant and tempo
 * factor per utterance ----------------------------------------------------------------------------------------------
 * y_length of world_b200_transform_*: the demo's formula (test.cpp:418-419) with the synthesis frame period
 *   fp = frame_period * time_scale (one product, rounded once):
 *   (int)((world_b200_frames(fs, x_length, frame_period) - 1) * fp / 1000.0 * fs) + 1
 * 0 when fp is not finite and > 0, or the length does not fit an int. */
int world_b200_transform_samples(int fs, int x_length, double frame_period, double time_scale);
/* x: n_utts rows of x_stride samples of `nbit` bits (DEVICE), as for world_b200_analyze_coded_batch (0 = doubles;
 * 8/16/24/32 = little-endian PCM); x_lengths HOST or NULL.  option selects the F0 method and carries its options and
 * those of CheapTrick and D4C; harvest_options / dio_options are NULL or one option per utterance of that F0 method
 * (HOST arrays of n_utts), with the rules of world_b200_analyze_batch_options / _dio_options.
 *   - f0_scale, spectral_ratio, time_scale: HOST arrays of n_utts, or NULL.  f0_scale and spectral_ratio change f0 and
 *     the spectral envelope as world_b200_modify_batch does (NULL skips that half).  Utterance u is synthesised with
 *     the frame period frame_period * time_scale[u] ms (NULL: 1.0): above 1 the speech is slower, below 1 faster;
 *     f0 and the envelopes are the same, only the frames are further apart.
 *   - y: [n_utts][y_stride] (DEVICE) of float64 for nbit_out 0, or int16 for nbit_out 16 (the pcm16 rule of
 *     world_b200_synthesis_coded_batch_pcm16); samples past an utterance's y_length are not written.  y_lengths (HOST,
 *     may be NULL) receives world_b200_transform_samples of each utterance.
 *   - Output: every row equals, bit for bit, world_b200_analyze_batch (full rows, the same options) ->
 *     world_b200_modify_batch (absent when f0_scale and spectral_ratio are both NULL) -> world_b200_synthesis_batch with
 *     frame_period * time_scale[u] and that y_length, for nbit_out 16 followed by the pcm16 rule.
 *   - The batch runs in utterance slices on the two internal streams of world_b200_analyze_batch; a slice's full rows
 *     live only from its analysis to its synthesis, so device memory does not grow with the batch.  The synthesis of
 *     one slice (whose time base is latency bound) runs beside the analysis of the next.  Synthesis reads its pulse
 *     counts back once per pass, so the host waits inside the call; the caller's stream is ordered after the work.
 *   - Validation, before any work is queued (WORLD_B200_EINVAL, world_b200_last_error() naming the first bad
 *     utterance; y is unchanged): what world_b200_analyze_coded_batch, world_b200_modify_batch and
 *     world_b200_synthesis_batch check, a time_scale that is not finite or not > 0, option->cheaptrick.fft_size outside
 *     Synthesis's powers of two in [16, 4096], an utterance of fewer than 2 frames or a y_length above y_stride, and an
 *     nbit_out other than 0 or 16.  n_utts 0 returns 0. */
int world_b200_transform_batch(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths,
                               int fs, const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                               const DioOption *dio_options, const double *f0_scale, const double *spectral_ratio,
                               const double *time_scale, int nbit_out, void *y, int y_stride, int *y_lengths);
/* The same for HOST x, y and y_lengths: utterance chunks of PCM are uploaded on one stream, transformed as above, and
 * their output rows downloaded on another, so only PCM crosses PCIe.  Whole rows of y are written: samples past an
 * utterance's y_length read 0.  Bit for bit equal to world_b200_transform_batch; pinned host buffers let the copies
 * run under the kernels.  Returns when the results are in y. */
int world_b200_transform_host(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths,
                              int fs, const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                              const DioOption *dio_options, const double *f0_scale, const double *spectral_ratio,
                              const double *time_scale, int nbit_out, void *y, int y_stride, int *y_lengths);
/* world_b200_transform_batch / world_b200_transform_host with per-utterance spectral options: cheaptrick_options and
 * d4c_options are HOST arrays of n_utts (either may be NULL: option->cheaptrick / option->d4c for every utterance).
 * Utterance u is analysed by CheapTrick with cheaptrick_options[u] and by D4C at the same fft_size, then modified and
 * synthesised at that size.  Every row equals, bit for bit, world_b200_cheaptrick_batch_options /
 * world_b200_d4c_batch_options (after the F0 stage of world_b200_analyze_batch) -> world_b200_modify_batch_options ->
 * world_b200_synthesis_batch_options with frame_period * time_scale[u].  Validation adds the rules of the stage calls
 * with options, and each utterance's fft_size within Synthesis's powers of two in [16, 4096]. */
int world_b200_transform_batch_spectral_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                                const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                                const HarvestOption *harvest_options, const DioOption *dio_options,
                                                const CheapTrickOption *cheaptrick_options,
                                                const D4COption *d4c_options, const double *f0_scale,
                                                const double *spectral_ratio, const double *time_scale, int nbit_out,
                                                void *y, int y_stride, int *y_lengths);
int world_b200_transform_host_spectral_options(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                               const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                               const HarvestOption *harvest_options, const DioOption *dio_options,
                                               const CheapTrickOption *cheaptrick_options,
                                               const D4COption *d4c_options, const double *f0_scale,
                                               const double *spectral_ratio, const double *time_scale, int nbit_out,
                                               void *y, int y_stride, int *y_lengths);
/* The voice transformation on a packed batch: utterances back to back in, transformed samples back to back out.
 * x_offsets is a HOST array of n_utts + 1 sample offsets with the rules of the packed analysis calls (above): x
 * holds nbit 0/8/16/24/32 samples, with byte offset = sample offset * nbit / 8.  Utterance u's output is samples
 * [y_offsets[u], y_offsets[u + 1]) of y, [Y] float64 (nbit_out 0) or int16 (nbit_out 16, the pcm16 rule), where
 * Y = y_offsets[n_utts] and
 *   y_offsets[0] = 0, y_offsets[u + 1] - y_offsets[u] =
 *     world_b200_transform_samples(fs, x_offsets[u + 1] - x_offsets[u], frame_period, time_scale ? time_scale[u] : 1)
 * with the F0 method's frame_period.  Every offset is 64-bit: Y may exceed 2^31.
 * world_b200_transform_packed_samples gives y_offsets (HOST, n_utts + 1) beforehand; EINVAL for bad offsets, a
 * time_scale that is not finite and > 0, or an utterance whose output length does not fit an int. */
int world_b200_transform_packed_samples(int fs, int n_utts, const long long *x_offsets, double frame_period,
                                        const double *time_scale, long long *y_offsets);
/* On DEVICE x and y.  The option arrays and factors are those of world_b200_transform_batch_spectral_options.
 *   - Output: utterance u's samples equal, bit for bit, row u of world_b200_transform_batch_spectral_options (or
 *     world_b200_transform_batch when both spectral option arrays are NULL) on the same utterances padded, with the
 *     same options and factors.  Samples [0, Y) of y are written and nothing else.  y_offsets (HOST, n_utts + 1, may be
 *     NULL) receives the sample offsets before any work is queued.
 *   - The batch runs in slices cut by their own lengths: a slice's rows are as long as its own longest utterance, so
 *     one long utterance does not shrink every slice.  Synthesis runs in packed passes.
 *   - Validation, before any work is queued (WORLD_B200_EINVAL, world_b200_last_error() naming the first bad
 *     utterance; y is unchanged): the padded call's rules (time_scale, at least 2 frames per utterance, Synthesis's FFT
 *     sizes, nbit_out, y given), the offset rules of the packed analysis calls, and an output length that does not fit
 *     an int.  n_utts 0 writes y_offsets[0] = 0 and returns 0. */
int world_b200_transform_packed(WorldB200 *ctx, const void *x, int nbit, int n_utts, const long long *x_offsets,
                                int fs, const WorldB200AnalysisOption *option, const HarvestOption *harvest_options,
                                const DioOption *dio_options, const CheapTrickOption *cheaptrick_options,
                                const D4COption *d4c_options, const double *f0_scale, const double *spectral_ratio,
                                const double *time_scale, int nbit_out, void *y, long long *y_offsets);
/* The same for HOST x and y: chunks of consecutive utterances go up as one copy of their samples and come back as one
 * copy of their output samples; no padding crosses PCIe.  Writes exactly Y samples, equal to
 * world_b200_transform_packed's; pinned host buffers let the copies run under the kernels.  Returns when the results
 * are in y. */
int world_b200_transform_host_packed(WorldB200 *ctx, const void *x, int nbit, int n_utts, const long long *x_offsets,
                                     int fs, const WorldB200AnalysisOption *option,
                                     const HarvestOption *harvest_options, const DioOption *dio_options,
                                     const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                     const double *f0_scale, const double *spectral_ratio, const double *time_scale,
                                     int nbit_out, void *y, long long *y_offsets);
/* world_b200_transform_packed / world_b200_transform_host_packed with pitch and formant curves in place of f0_scale and
 * spectral_ratio (time_scale stays one factor per utterance).  The curves are on the analysis frame grid: [F] frames at
 * the offsets world_b200_packed_frames(fs, n_utts, x_offsets, frame_period) gives for the F0 method's frame_period;
 * DEVICE arrays for world_b200_transform_packed_curves, HOST arrays for world_b200_transform_host_packed_curves (each
 * chunk's curve frames go up as one copy beside its samples).  Either may be NULL.  Every utterance's output equals,
 * bit for bit, world_b200_analyze_packed -> world_b200_modify_curves_packed -> world_b200_synthesis_packed at
 * frame_period * time_scale[u]; with constant curves it equals world_b200_transform_packed with those factors.
 * Validation adds the per-frame rules of world_b200_modify_curves to the packed transform's, before any work is queued;
 * the device call checks its curves with one kernel and one synchronisation. */
int world_b200_transform_packed_curves(WorldB200 *ctx, const void *x, int nbit, int n_utts, const long long *x_offsets,
                                       int fs, const WorldB200AnalysisOption *option,
                                       const HarvestOption *harvest_options, const DioOption *dio_options,
                                       const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                       const double *f0_curve, const double *spectral_ratio_curve,
                                       const double *time_scale, int nbit_out, void *y, long long *y_offsets);
int world_b200_transform_host_packed_curves(WorldB200 *ctx, const void *x, int nbit, int n_utts,
                                            const long long *x_offsets, int fs, const WorldB200AnalysisOption *option,
                                            const HarvestOption *harvest_options, const DioOption *dio_options,
                                            const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                            const double *f0_curve, const double *spectral_ratio_curve,
                                            const double *time_scale, int nbit_out, void *y, long long *y_offsets);

#ifdef __cplusplus
}
#endif
#endif /* WORLD_B200_H_ */
