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
 *     the context's stream (world_b200_set_stream); they do not synchronise.  The *_host
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
                                  (e.g. f0 below the floor implied by fft_size); see message  */

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
/* Synchronises and releases the device memory the context keeps between calls (scratch arena and the
 * staging buffers of the *_host pipelines); the next call allocates again. */
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

/* Test hook: forward real FFT of n = 2^k doubles (4 <= n <= 8192) with the library's shared-memory
 * FFT; out_dev receives n/2+1 interleaved complex values (n + 2 doubles).  DEVICE pointers. */
int world_b200_rfft_test(WorldB200 *ctx, const double *x_dev, int n, double *out_dev);
/* same, through the self-sorting padded FFT the frame kernels use since round 2 */
int world_b200_sfft_test(WorldB200 *ctx, const double *x_dev, int n, double *out_dev);

/* Test hook: first n_draws values of the reference's randn() stream (matlabfunctions.cpp:237-264)
 * as raw 32-bit sums (value = sum / 2^28 - 6) into a DEVICE buffer of n_draws uint32. */
int world_b200_randn_stream(WorldB200 *ctx, unsigned n_draws, unsigned *out_dev);

/* int(1000.0 * x_length / fs / frame_period) + 1 */
int world_b200_frames(int fs, int x_length, double frame_period);

/* ---- batched stages, device pointers -------------------------------------------------- */
/* Dio() over a batch (dio.h:38).  Writes time_axis and f0 rows of world_b200_frames() entries. */
int world_b200_dio_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                         const int *x_lengths, int fs, const DioOption *option,
                         double *time_axis, double *f0, int f0_stride);
/* Harvest() over a batch (harvest.h:35). */
int world_b200_harvest_batch(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                             const int *x_lengths, int fs, const HarvestOption *option,
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

/* {Dio+StoneMask | Harvest} -> CheapTrick -> D4C for n_utts host waveforms; outputs are host
 * arrays laid out as described above.  Input upload, compute and result download are pipelined
 * over utterance chunks.  Any output pointer may be NULL to skip its download.  Whole padded rows
 * are downloaded: frames beyond an utterance's own count come back as zeros. */
int world_b200_analyze_host(WorldB200 *ctx, const double *x, int n_utts, int x_stride,
                            const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                            double *time_axis, double *f0, int f0_stride, double *spectrogram,
                            double *aperiodicity);

/* The same chain with the ingest and the codec fused in on the device: x holds samples of `nbit`
 * bits (0 = doubles as above; 8/16/24/32 = little-endian PCM as in a WAV data chunk), and the
 * results that cross PCIe are the coded rows -- coded_spectral_envelope [n][f0_stride]
 * [number_of_dimensions], coded_aperiodicity [n][f0_stride][GetNumberOfAperiodicities(fs)] -- about
 * 8.4 times (16 kHz, 60 dimensions) fewer device-to-host bytes than the full rows. */
int world_b200_analyze_coded_host(WorldB200 *ctx, const void *x, int nbit, int n_utts, int x_stride,
                                  const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                  int number_of_dimensions, double *time_axis, double *f0, int f0_stride,
                                  double *coded_spectral_envelope, double *coded_aperiodicity);

#ifdef __cplusplus
}
#endif
#endif /* WORLD_B200_H_ */
