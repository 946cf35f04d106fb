// wb_host.cu -- host-pointer entry points built on the device-pointer ABI:
//   * world_b200_analyze_host(): {Dio+StoneMask | Harvest} -> CheapTrick -> D4C for N host
//     waveforms, upload / compute / download pipelined over utterance chunks on three streams;
//   * world_b200_synthesis_coded_host(): the way back, f0 + coded rows -> waveforms or 16-bit PCM,
//     pipelined the same way;
//   * the reference's own single-utterance functions (Dio, Harvest, StoneMask, CheapTrick, D4C;
//     src/world/*.h) as n_utts = 1 batches on a lazily created process-wide context, so existing
//     callers relink unchanged.  They keep the reference's `void` signature; failures are
//     reported on stderr and leave the outputs zero-filled.
#include "wb_internal.h"
#include "../../include/world_b200.h"
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <memory>
#include <mutex>
#include <chrono>

using namespace wb;

namespace wb {
// wb_api.cu: checks of per-utterance F0 options for a chain, and the chain's F0 stage
int check_chain_f0_options(Ctx *c, const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                           const DioOption *dio_options, int n, int fs, const char *who);
int run_f0_stage(WorldB200 *h, const double *x, int m, int x_stride, const int *x_lengths, int fs,
                 const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options, const DioOption *dio_options,
                 const int *f0_lengths, double *time_axis, double *f0, int f0_stride);
}  // namespace wb

namespace {

struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
};

int ensure(Ctx *ctx, DevBuf *b, size_t bytes) {   // pooled: kept by the context between calls
  if (bytes <= b->cap) return 0;
  pool_release(ctx, b->p);
  b->p = pool_acquire(ctx, bytes);
  b->cap = b->p ? bytes : 0;
  return b->p ? 0 : WORLD_B200_ENOMEM;
}

Ctx *ctx_of(WorldB200 *h) { return reinterpret_cast<Ctx *>(h); }  // Ctx is the first member

}  // namespace

namespace {

// One pipeline for both host entry points.  nbit == 0: x holds doubles; otherwise little-endian PCM that
// is widened on the device (row f3).  dims == 0: the full spectrogram / aperiodicity rows go back to the
// host; dims > 0: they stay on the device and only their coded rows (row f2) are downloaded.
//
// Two granularities.  The F0 stage runs on OUTER chunks (default 512 utterances): its per-utterance
// kernels (contour tracking, smoothing, decimation) are latency bound -- one launch costs the same
// for 96 or 500 utterances -- so few large launches beat many small ones.  CheapTrick / D4C (/ codec) run
// on SUB-chunks (default 128 utterances) whose rows start their trip over PCIe as soon as they exist: the
// un-overlapped tail is one sub-chunk.  Result buffers form a ring two outer chunks deep, so downloads
// may lag behind the frame kernels and catch up under the next outer chunk's F0 stage.  Streams: s_in
// (uploads), the context's stream (all kernels), s_out (downloads); events order buffer reuse.
// harvest_options / dio_options: nullptr, or one option per utterance (checked by the caller, at most one of the two);
// the outer chunks split the array.
int analyze_pipeline(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths, int fs,
                     const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                     const DioOption *dio_options, int dims, double *time_axis, double *f0, int f0_stride,
                     double *out_sp, double *out_ap) {
  Ctx *ctx = ctx_of(h);
  const int bins = opt->cheaptrick.fft_size / 2 + 1;
  const int n_ap = GetNumberOfAperiodicities(fs);
  const size_t in_bytes = nbit ? (size_t)(nbit / 8) : 8;
  const size_t sp_row = dims ? (size_t)dims : (size_t)bins, ap_row = dims ? (size_t)n_ap : (size_t)bins;
  const double frame_period =
      opt->f0_method == WORLD_B200_F0_HARVEST ? opt->harvest.frame_period : opt->dio.frame_period;
  const bool want_sp = out_sp != nullptr, want_ap = out_ap != nullptr && (!dims || n_ap > 0);
  if (n_utts == 0) return 0;
  // coded mode: the frame kernels write the coded rows themselves (world_b200_cheaptrick_coded_batch /
  // world_b200_d4c_coded_batch); WB_CODEC_UNFUSED=1 keeps round 1's full rows + codec kernels for A/B runs
  const bool unfused = dims && getenv("WB_CODEC_UNFUSED") != nullptr;

  int sub = 128, outer = 512;
  if (const char *e = getenv("WB_HOST_SUB")) sub = atoi(e) > 0 ? atoi(e) : sub;
  if (const char *e = getenv("WB_HOST_CHUNK")) outer = atoi(e) > 0 ? atoi(e) : outer;
  sub = imin(sub, n_utts);
  // a third of the scratch budget for this pipeline's own buffers: two outer sets + the result ring
  const size_t third = ctx->scratch_budget / 3;
  const size_t per_outer = (size_t)x_stride * (in_bytes + (nbit ? 8 : 0)) + (size_t)f0_stride * 16;
  const size_t per_sub_out = (size_t)f0_stride * ((want_sp ? sp_row : 0) + (want_ap ? ap_row : 0)) * 8;
  const size_t per_sub_raw = (size_t)f0_stride * ((want_sp ? bins : 0) + (want_ap ? bins : 0)) * 8;
  outer = imin(outer, (int)dmax((double)sub, (double)(third / 3) / (double)(2 * per_outer)));
  outer = imax(sub, outer / sub * sub);
  outer = imin(outer, (n_utts + sub - 1) / sub * sub);
  const int subs_per_outer = outer / sub;
  const double ring_budget = (double)third - (double)imin(n_utts, outer) * 2.0 * (double)per_outer -
                             (unfused ? (double)sub * (double)per_sub_raw : 0.0);
  int ring = 2 * subs_per_outer;
  if (per_sub_out > 0)
    ring = imax(2, imin(ring, (int)dmax(0.0, ring_budget / ((double)sub * (double)per_sub_out))));
  ring = imin(ring, (n_utts + sub - 1) / sub);
  if (ring < 1) ring = 1;

#ifndef WB_EMU
  cudaStream_t s_compute = ctx->stream, s_in = nullptr, s_out = nullptr;
  if (cudaStreamCreateWithFlags(&s_in, cudaStreamNonBlocking) != cudaSuccess) {
    ctx->last_error = "cudaStreamCreate failed";
    cudaGetLastError();
    return WORLD_B200_ECUDA;
  }
  if (cudaStreamCreateWithFlags(&s_out, cudaStreamNonBlocking) != cudaSuccess) {
    ctx->last_error = "cudaStreamCreate failed";
    cudaGetLastError();
    cudaStreamDestroy(s_in);
    return WORLD_B200_ECUDA;
  }
  cudaEvent_t ev_in[2], ev_cdone[2], ev_f0[2], ev_tf[2], ev_start;
  bool ev_ok = cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming) == cudaSuccess;
  for (int i = 0; i < 2; ++i) {
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_in[i], cudaEventDisableTiming) == cudaSuccess;
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_cdone[i], cudaEventDisableTiming) == cudaSuccess;
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_f0[i], cudaEventDisableTiming) == cudaSuccess;
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_tf[i], cudaEventDisableTiming) == cudaSuccess;
  }
  std::vector<cudaEvent_t> ev_sub_done(ring), ev_sub_out(ring);
  for (int i = 0; i < ring; ++i) {
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_sub_done[i], cudaEventDisableTiming) == cudaSuccess;
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_sub_out[i], cudaEventDisableTiming) == cudaSuccess;
  }
  if (!ev_ok) {   // (events created so far are released with the process; this only happens when the driver is out of resources)
    ctx->last_error = "cudaEventCreate failed";
    cudaGetLastError();
    cudaStreamDestroy(s_in);
    cudaStreamDestroy(s_out);
    return WORLD_B200_ECUDA;
  }
#endif
  // WB_HOST_TRACE=1: timeline of this call on stderr (timing events on the three streams + host clock)
  const bool trace = getenv("WB_HOST_TRACE") != nullptr;
  struct Mark { const char *what; int idx; double host_ms; void *ev; };
  std::vector<Mark> marks;
  const auto t_host0 = std::chrono::steady_clock::now();
  auto mark = [&](const char *what, int idx, void *stream) {
    if (!trace) return;
    Mark m{what, idx, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count(), nullptr};
#ifndef WB_EMU
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, (cudaStream_t)stream);
    m.ev = e;
#else
    (void)stream;
#endif
    marks.push_back(m);
  };
#ifndef WB_EMU
  mark("start", 0, s_compute);
  // the uploads start after the work already on the context's stream: a pooled buffer released by a stream-ordered
  // call (the PCM buffer of world_b200_analyze_coded_batch) may still be read there
  cudaEventRecord(ev_start, s_compute);
  cudaStreamWaitEvent(s_in, ev_start, 0);
#endif
  DevBuf din[2], dx[2], dt[2], df[2];
  const int raw_slots = dims ? (unfused ? 1 : 0) : ring;   // unfused coded mode: the full rows are consumed on the same stream
  std::vector<DevBuf> dsp(raw_slots), dap(raw_slots), dcs(dims ? ring : 0), dca(dims ? ring : 0);
  int rc = 0;
  const int n_outer_bufs = n_utts > outer ? 2 : 1;
  for (int i = 0; i < n_outer_bufs && !rc; ++i) {
    rc = ensure(ctx, &din[i], (size_t)outer * x_stride * in_bytes);
    if (!rc && nbit) rc = ensure(ctx, &dx[i], (size_t)outer * x_stride * 8);
    if (!rc) rc = ensure(ctx, &dt[i], (size_t)outer * f0_stride * 8);
    if (!rc) rc = ensure(ctx, &df[i], (size_t)outer * f0_stride * 8);
  }
  for (int i = 0; i < raw_slots && !rc; ++i) {
    if (want_sp) rc = ensure(ctx, &dsp[i], (size_t)sub * f0_stride * bins * 8);
    if (!rc && want_ap) rc = ensure(ctx, &dap[i], (size_t)sub * f0_stride * bins * 8);
  }
  for (int i = 0; i < (dims ? ring : 0) && !rc; ++i) {
    if (want_sp) rc = ensure(ctx, &dcs[i], (size_t)sub * f0_stride * sp_row * 8);
    if (!rc && want_ap) rc = ensure(ctx, &dca[i], (size_t)sub * f0_stride * ap_row * 8);
  }
  std::vector<int> flen(n_utts);
  for (int i = 0; i < n_utts && !rc; ++i) {
    flen[i] = world_b200_frames(fs, x_lengths ? x_lengths[i] : x_stride, frame_period);
    if (flen[i] > f0_stride) { ctx->last_error = "f0_stride too small"; rc = WORLD_B200_EINVAL; }
  }
  int it = 0, g = 0;   // outer chunk counter, global sub-chunk counter
  for (int u0 = 0; u0 < n_utts && !rc; u0 += outer, ++it) {
    const int n = imin(outer, n_utts - u0);
    const int s = it & 1;
    const int *xl = x_lengths ? x_lengths + u0 : nullptr;
    const int *fl = flen.data() + u0;
    const size_t fsz = (size_t)n * f0_stride;
    const unsigned char *src = (const unsigned char *)x + (size_t)u0 * x_stride * in_bytes;
#ifndef WB_EMU
    if (it >= 2) cudaStreamWaitEvent(s_in, ev_cdone[s], 0);   // kernels of outer chunk it-2 read din[s] / dx[s]
    cudaMemcpyAsync(din[s].p, src, (size_t)n * x_stride * in_bytes, cudaMemcpyHostToDevice, s_in);
    cudaEventRecord(ev_in[s], s_in);
    mark("h2d_done", it, s_in);
    cudaStreamWaitEvent(s_compute, ev_in[s], 0);
    if (it >= 2) cudaStreamWaitEvent(s_compute, ev_tf[s], 0);  // time_axis / f0 of it-2 are on the host
    mark("f0_begin", it, s_compute);
#else
    memcpy(din[s].p, src, (size_t)n * x_stride * in_bytes);
#endif
    if (nbit) rc = world_b200_pcm_to_double_batch(h, din[s].p, nbit, n, x_stride, xl, (double *)dx[s].p);
    if (rc) break;
    dev_memset(ctx, dt[s].p, 0, fsz * 8);
    dev_memset(ctx, df[s].p, 0, fsz * 8);
    const double *xd = (const double *)(nbit ? dx[s].p : din[s].p);
    double *td = (double *)dt[s].p, *fd = (double *)df[s].p;
    rc = run_f0_stage(h, xd, n, x_stride, xl, fs, opt, harvest_options ? harvest_options + u0 : nullptr,
                      dio_options ? dio_options + u0 : nullptr, fl, td, fd, f0_stride);
    if (rc) break;
#ifndef WB_EMU
    cudaEventRecord(ev_f0[s], s_compute);
    mark("f0_end", it, s_compute);
    cudaStreamWaitEvent(s_out, ev_f0[s], 0);
    if (time_axis) cudaMemcpyAsync(time_axis + (size_t)u0 * f0_stride, td, fsz * 8, cudaMemcpyDeviceToHost, s_out);
    if (f0) cudaMemcpyAsync(f0 + (size_t)u0 * f0_stride, fd, fsz * 8, cudaMemcpyDeviceToHost, s_out);
    cudaEventRecord(ev_tf[s], s_out);
#else
    if (time_axis) memcpy(time_axis + (size_t)u0 * f0_stride, td, fsz * 8);
    if (f0) memcpy(f0 + (size_t)u0 * f0_stride, fd, fsz * 8);
#endif
    // Sub-chunk size.  A sub-chunk's rows go to the host while the next one is computed, and in the full-row mode a
    // sub-chunk takes ~12 % longer to download than to compute: after the LAST outer chunk the copy engine is the
    // critical path, finishing (first sub-chunk's compute + every download) after the chunk's Harvest -- ~50 ms behind
    // the kernels of a 850 ms step at 1024 x 10 s with sub-chunks of 128.  Quarter-size sub-chunks there start the
    // downloads earlier and leave a shorter last one (~25 ms behind).  WB_HOST_TAPER=0 disables it.
    const bool taper = !dims && u0 + outer >= n_utts && !(getenv("WB_HOST_TAPER") && atoi(getenv("WB_HOST_TAPER")) == 0);
    int taper_min = 16;   // (WB_HOST_TAPER_MIN: tests exercise the path with a handful of utterances)
    if (const char *e = getenv("WB_HOST_TAPER_MIN")) taper_min = imax(1, atoi(e));
    int taper_div = 4;
    if (const char *e = getenv("WB_HOST_TAPER_DIV")) taper_div = imax(1, atoi(e));
    const int sub_here = taper ? imax(imin(sub, taper_min), sub / taper_div) : sub;
    for (int v0 = 0; v0 < n && !rc && (want_sp || want_ap); v0 += sub_here, ++g) {
      const int m = imin(sub_here, n - v0);
      const int slot = g % ring, rslot = dims ? 0 : slot;
      const int *sxl = xl ? xl + v0 : nullptr;
      const int *sfl = fl + v0;
      const size_t ssz = (size_t)m * f0_stride;
      const double *sx = xd + (size_t)v0 * x_stride, *st = td + (size_t)v0 * f0_stride, *sf = fd + (size_t)v0 * f0_stride;
#ifndef WB_EMU
      if (g >= ring) cudaStreamWaitEvent(s_compute, ev_sub_out[slot], 0);   // the slot's previous rows are on the host
#endif
      // whole padded rows are downloaded: frames beyond an utterance's length read as zero on the host
      bool ragged = false;
      for (int i = 0; i < m; ++i) ragged = ragged || sfl[i] != f0_stride;
      if (ragged) {
        if (!dims && want_sp) dev_memset(ctx, dsp[rslot].p, 0, ssz * bins * 8);
        if (!dims && want_ap) dev_memset(ctx, dap[rslot].p, 0, ssz * bins * 8);
        if (dims && want_sp) dev_memset(ctx, dcs[slot].p, 0, ssz * sp_row * 8);
        if (dims && want_ap) dev_memset(ctx, dca[slot].p, 0, ssz * ap_row * 8);
      }
      if (dims && !unfused) {
        if (want_sp)
          rc = world_b200_cheaptrick_coded_batch(h, sx, m, x_stride, sxl, fs, st, sf, sfl, f0_stride, &opt->cheaptrick,
                                                 dims, (double *)dcs[slot].p);
        if (!rc && want_ap)
          rc = world_b200_d4c_coded_batch(h, sx, m, x_stride, sxl, fs, st, sf, sfl, f0_stride,
                                          opt->cheaptrick.fft_size, &opt->d4c, (double *)dca[slot].p);
      } else {
        if (want_sp)
          rc = world_b200_cheaptrick_batch(h, sx, m, x_stride, sxl, fs, st, sf, sfl, f0_stride, &opt->cheaptrick,
                                           (double *)dsp[rslot].p);
        if (!rc && want_ap)
          rc = world_b200_d4c_batch(h, sx, m, x_stride, sxl, fs, st, sf, sfl, f0_stride, opt->cheaptrick.fft_size,
                                    &opt->d4c, (double *)dap[rslot].p);
        if (!rc && dims && want_sp)
          rc = world_b200_code_spectral_envelope_batch(h, (const double *)dsp[0].p, m, sfl, f0_stride, fs,
                                                       opt->cheaptrick.fft_size, dims, (double *)dcs[slot].p);
        if (!rc && dims && want_ap)
          rc = world_b200_code_aperiodicity_batch(h, (const double *)dap[0].p, m, sfl, f0_stride, fs,
                                                  opt->cheaptrick.fft_size, (double *)dca[slot].p);
      }
      if (rc) break;
      const void *sp_src = dims ? dcs[slot].p : dsp[rslot].p, *ap_src = dims ? dca[slot].p : dap[rslot].p;
      const size_t row0 = (size_t)(u0 + v0) * f0_stride;
#ifndef WB_EMU
      cudaEventRecord(ev_sub_done[slot], s_compute);
      mark("sub_end", g, s_compute);
      cudaStreamWaitEvent(s_out, ev_sub_done[slot], 0);
      if (want_sp) cudaMemcpyAsync(out_sp + row0 * sp_row, sp_src, ssz * sp_row * 8, cudaMemcpyDeviceToHost, s_out);
      if (want_ap) cudaMemcpyAsync(out_ap + row0 * ap_row, ap_src, ssz * ap_row * 8, cudaMemcpyDeviceToHost, s_out);
      cudaEventRecord(ev_sub_out[slot], s_out);
      mark("d2h_end", g, s_out);
#else
      if (want_sp) memcpy(out_sp + row0 * sp_row, sp_src, ssz * sp_row * 8);
      if (want_ap) memcpy(out_ap + row0 * ap_row, ap_src, ssz * ap_row * 8);
#endif
    }
#ifndef WB_EMU
    cudaEventRecord(ev_cdone[s], s_compute);
#endif
  }
#ifndef WB_EMU
  const double issued_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count();
  // copies and memsets above are not checked one by one: a failure is sticky and surfaces here
  cudaError_t e_sync = cudaStreamSynchronize(s_in);
  if (e_sync == cudaSuccess) e_sync = cudaStreamSynchronize(s_compute);
  if (e_sync == cudaSuccess) e_sync = cudaStreamSynchronize(s_out);
  if (e_sync != cudaSuccess && !rc) { ctx->last_error = std::string("analyze pipeline: ") + cudaGetErrorString(e_sync); rc = WORLD_B200_ECUDA; }
  if (trace && !marks.empty()) {
    const double done_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count();
    fprintf(stderr, "[wb trace] outer %d sub %d ring %d n %d: all work issued at %.1f ms, finished at %.1f ms (host clock)\n",
            outer, sub, ring, n_utts, issued_ms, done_ms);
    for (size_t i = 1; i < marks.size(); ++i) {
      float gpu_ms = 0.f;
      cudaEventElapsedTime(&gpu_ms, (cudaEvent_t)marks[0].ev, (cudaEvent_t)marks[i].ev);
      fprintf(stderr, "[wb trace] %-9s %3d  issued %8.1f  gpu %8.1f\n", marks[i].what, marks[i].idx, marks[i].host_ms, gpu_ms);
    }
    for (auto &m : marks) cudaEventDestroy((cudaEvent_t)m.ev);
  }
  for (int i = 0; i < 2; ++i) {
    cudaEventDestroy(ev_in[i]); cudaEventDestroy(ev_cdone[i]); cudaEventDestroy(ev_f0[i]); cudaEventDestroy(ev_tf[i]);
  }
  for (int i = 0; i < ring; ++i) { cudaEventDestroy(ev_sub_done[i]); cudaEventDestroy(ev_sub_out[i]); }
  cudaEventDestroy(ev_start);
  cudaStreamDestroy(s_in);
  cudaStreamDestroy(s_out);
  if (!rc) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { ctx->last_error = cudaGetErrorString(e); rc = WORLD_B200_ECUDA; }
  }
#endif
  for (int i = 0; i < 2; ++i) { pool_release(ctx, din[i].p); pool_release(ctx, dx[i].p); pool_release(ctx, dt[i].p); pool_release(ctx, df[i].p); }
  for (auto &b : dsp) pool_release(ctx, b.p);
  for (auto &b : dap) pool_release(ctx, b.p);
  for (auto &b : dcs) pool_release(ctx, b.p);
  for (auto &b : dca) pool_release(ctx, b.p);
  if (!rc) rc = world_b200_synchronize(h);
  return rc;
}

}  // namespace

namespace {

// Synthesis from coded rows for host arrays: utterance chunks, uploads on s_in, synthesis_run on the context's stream,
// downloads on s_out.  Inputs (f0 + coded rows) are double-buffered, outputs go through a ring of `ring` chunk slots;
// events order the reuse of both.  synthesis_run synchronises the context's stream once per pass (its pulse counts),
// so the upload of chunk k+1 is enqueued before synthesis_run is called for chunk k: it then runs under chunk k's
// kernels instead of after the host has waited for them.  A chunk is one pass of synthesis_run: a longer chunk would
// hold its download until all its passes were done, and a shorter one would pay the pass's fixed cost more often
// (syn_timebase_kernel's sequential phase sum over each utterance takes about as long for a few utterances as for a
// pass of hundreds; at 1024 x 10 s, 16 kHz, chunks of 128 utterances made the call slower than the serial path).  Two
// input sets and the output ring stay within a third of the scratch budget.  `lens` holds the checked lengths
// (synthesis_lengths).
int synthesis_pipeline(WorldB200 *h, CodedRows *coded, int lg, const double *f0, const int *f0_lengths, int n_utts,
                       int f0_stride, int fft_size, double frame_period, int fs, const int *y_lengths, int y_stride,
                       const int *lens, int nbit, void *y) {
  Ctx *ctx = ctx_of(h);
  const int dims = coded->tsp.dims, n_ap = coded->tap.dims;
  const double *h_sp = coded->sp, *h_ap = coded->ap;
  const size_t out_bytes = nbit ? 2 : 8;
  const size_t per_in = (size_t)f0_stride * (1 + dims + n_ap) * 8, per_out = (size_t)y_stride * out_bytes;
  int max_y = 0;
  for (int i = 0; i < n_utts; ++i) max_y = imax(max_y, lens[n_utts + i]);
  const SynthesisSizing sz(ctx, coded, fft_size, f0_stride, y_stride, max_y, fs);
  int ring = 3;
  const size_t third = ctx->scratch_budget / 3;
  int chunk = imax(1, sz.fit(sz.nominal_cap));
  chunk = imin(chunk, (int)dmax(1.0, (double)third / (double)(2 * per_in + ring * per_out)));
  chunk = balanced_chunk(n_utts, chunk);
  const int n_chunks = (n_utts + chunk - 1) / chunk;
  ring = imin(ring, n_chunks);
  ArenaPlan in_plan;
  const size_t o_f0 = in_plan.add((size_t)chunk * f0_stride * 8);
  const size_t o_sp = in_plan.add((size_t)chunk * f0_stride * dims * 8);
  const size_t o_ap = in_plan.add((size_t)chunk * f0_stride * n_ap * 8);

#ifndef WB_EMU
  cudaStream_t s_compute = ctx->stream, s_in = nullptr, s_out = nullptr;
  if (cudaStreamCreateWithFlags(&s_in, cudaStreamNonBlocking) != cudaSuccess) {
    ctx->last_error = "cudaStreamCreate failed";
    cudaGetLastError();
    return WORLD_B200_ECUDA;
  }
  if (cudaStreamCreateWithFlags(&s_out, cudaStreamNonBlocking) != cudaSuccess) {
    ctx->last_error = "cudaStreamCreate failed";
    cudaGetLastError();
    cudaStreamDestroy(s_in);
    return WORLD_B200_ECUDA;
  }
  cudaEvent_t ev_in[2], ev_cdone[2], ev_start;
  std::vector<cudaEvent_t> ev_out(ring);
  bool ev_ok = cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming) == cudaSuccess;
  for (int i = 0; i < 2; ++i) {
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_in[i], cudaEventDisableTiming) == cudaSuccess;
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_cdone[i], cudaEventDisableTiming) == cudaSuccess;
  }
  for (int i = 0; i < ring; ++i)
    ev_ok = ev_ok && cudaEventCreateWithFlags(&ev_out[i], cudaEventDisableTiming) == cudaSuccess;
  if (!ev_ok) {   // (as in analyze_pipeline: events created so far are released with the process)
    ctx->last_error = "cudaEventCreate failed";
    cudaGetLastError();
    cudaStreamDestroy(s_in);
    cudaStreamDestroy(s_out);
    return WORLD_B200_ECUDA;
  }
#endif
  // WB_HOST_TRACE=1: timeline of this call on stderr (timing events on the three streams + host clock)
  const bool trace = getenv("WB_HOST_TRACE") != nullptr;
  struct Mark { const char *what; int idx; double host_ms; void *ev; };
  std::vector<Mark> marks;
  const auto t_host0 = std::chrono::steady_clock::now();
  auto mark = [&](const char *what, int idx, void *stream) {
    if (!trace) return;
    Mark m{what, idx, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count(), nullptr};
#ifndef WB_EMU
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, (cudaStream_t)stream);
    m.ev = e;
#else
    (void)stream;
#endif
    marks.push_back(m);
  };
#ifndef WB_EMU
  mark("start", 0, s_compute);
  // the uploads start after the work already on the context's stream: a pooled buffer released by a stream-ordered
  // call may still be read there
  cudaEventRecord(ev_start, s_compute);
  cudaStreamWaitEvent(s_in, ev_start, 0);
#endif
  DevBuf din[2];
  std::vector<DevBuf> dout(ring);
  int rc = 0;
  for (int i = 0; i < (n_chunks > 1 ? 2 : 1) && !rc; ++i) rc = ensure(ctx, &din[i], in_plan.total);
  for (int i = 0; i < ring && !rc; ++i) rc = ensure(ctx, &dout[i], (size_t)chunk * per_out);

  // chunk k's f0 and coded rows into din[k & 1]
  auto upload = [&](int k) {
    const int u0 = k * chunk, m = imin(chunk, n_utts - u0);
    const size_t frames = (size_t)m * f0_stride, row0 = (size_t)u0 * f0_stride;
    unsigned char *d = (unsigned char *)din[k & 1].p;
#ifndef WB_EMU
    if (k >= 2) cudaStreamWaitEvent(s_in, ev_cdone[k & 1], 0);   // the kernels of chunk k-2 have read din[k & 1]
    cudaMemcpyAsync(d + o_f0, f0 + row0, frames * 8, cudaMemcpyHostToDevice, s_in);
    cudaMemcpyAsync(d + o_sp, h_sp + row0 * dims, frames * dims * 8, cudaMemcpyHostToDevice, s_in);
    if (n_ap) cudaMemcpyAsync(d + o_ap, h_ap + row0 * n_ap, frames * n_ap * 8, cudaMemcpyHostToDevice, s_in);
    cudaEventRecord(ev_in[k & 1], s_in);
    mark("h2d_done", k, s_in);
#else
    memcpy(d + o_f0, f0 + row0, frames * 8);
    memcpy(d + o_sp, h_sp + row0 * dims, frames * dims * 8);
    if (n_ap) memcpy(d + o_ap, h_ap + row0 * n_ap, frames * n_ap * 8);
#endif
  };
  if (!rc) upload(0);
  for (int k = 0; k < n_chunks && !rc; ++k) {
    const int u0 = k * chunk, m = imin(chunk, n_utts - u0), s = k & 1, slot = k % ring;
    if (k + 1 < n_chunks) upload(k + 1);
    unsigned char *d = (unsigned char *)din[s].p;
#ifndef WB_EMU
    cudaStreamWaitEvent(s_compute, ev_in[s], 0);
    if (k >= ring) cudaStreamWaitEvent(s_compute, ev_out[slot], 0);   // the slot's previous chunk is on the host
    mark("syn_begin", k, s_compute);
#endif
    // whole padded rows are downloaded: samples beyond an utterance's length read as zero on the host
    bool ragged = false;
    for (int i = 0; i < m; ++i) ragged = ragged || lens[n_utts + u0 + i] != y_stride;
    if (ragged) rc = dev_memset(ctx, dout[slot].p, 0, (size_t)m * per_out);
    coded->sp = (const double *)(d + o_sp);
    coded->ap = n_ap ? (const double *)(d + o_ap) : nullptr;
    if (!rc)
      rc = synthesis_run(ctx, (const double *)(d + o_f0), f0_lengths ? f0_lengths + u0 : nullptr, m, f0_stride, nullptr,
                         nullptr, coded, fft_size, lg, frame_period, fs, y_lengths ? y_lengths + u0 : nullptr, y_stride,
                         dout[slot].p, nbit);
    if (rc) break;
    unsigned char *dst = (unsigned char *)y + (size_t)u0 * per_out;
#ifndef WB_EMU
    cudaEventRecord(ev_cdone[s], s_compute);   // behind chunk k's overlap kernel
    mark("syn_end", k, s_compute);
    cudaStreamWaitEvent(s_out, ev_cdone[s], 0);
    cudaMemcpyAsync(dst, dout[slot].p, (size_t)m * per_out, cudaMemcpyDeviceToHost, s_out);
    cudaEventRecord(ev_out[slot], s_out);
    mark("d2h_end", k, s_out);
#else
    memcpy(dst, dout[slot].p, (size_t)m * per_out);
#endif
  }
  coded->sp = h_sp;
  coded->ap = h_ap;
  const double issued_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count();
#ifndef WB_EMU
  // copies and memsets above are not checked one by one: a failure is sticky and surfaces here
  cudaError_t e_sync = cudaStreamSynchronize(s_in);
  if (e_sync == cudaSuccess) e_sync = cudaStreamSynchronize(s_compute);
  if (e_sync == cudaSuccess) e_sync = cudaStreamSynchronize(s_out);
  if (e_sync != cudaSuccess && !rc) { ctx->last_error = std::string("synthesis pipeline: ") + cudaGetErrorString(e_sync); rc = WORLD_B200_ECUDA; }
#endif
  if (trace) {
    const double done_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count();
    fprintf(stderr, "[wb trace] synthesis chunk %d chunks %d ring %d n %d nbit %d: all work issued at %.1f ms, "
            "finished at %.1f ms (host clock)\n", chunk, n_chunks, ring, n_utts, nbit, issued_ms, done_ms);
#ifndef WB_EMU
    for (size_t i = 1; i < marks.size(); ++i) {
      float gpu_ms = 0.f;
      cudaEventElapsedTime(&gpu_ms, (cudaEvent_t)marks[0].ev, (cudaEvent_t)marks[i].ev);
      fprintf(stderr, "[wb trace] %-9s %3d  issued %8.1f  gpu %8.1f\n", marks[i].what, marks[i].idx, marks[i].host_ms, gpu_ms);
    }
    for (auto &m : marks) cudaEventDestroy((cudaEvent_t)m.ev);
#endif
  }
#ifndef WB_EMU
  for (int i = 0; i < 2; ++i) { cudaEventDestroy(ev_in[i]); cudaEventDestroy(ev_cdone[i]); }
  for (int i = 0; i < ring; ++i) cudaEventDestroy(ev_out[i]);
  cudaEventDestroy(ev_start);
  cudaStreamDestroy(s_in);
  cudaStreamDestroy(s_out);
  if (!rc) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { ctx->last_error = cudaGetErrorString(e); rc = WORLD_B200_ECUDA; }
  }
#endif
  for (int i = 0; i < 2; ++i) pool_release(ctx, din[i].p);
  for (auto &b : dout) pool_release(ctx, b.p);
  if (!rc) rc = world_b200_synchronize(h);
  return rc;
}

}  // namespace

extern "C" int world_b200_synthesis_coded_host(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts,
                                               int f0_stride, const double *coded_spectral_envelope,
                                               int number_of_dimensions, const double *coded_aperiodicity,
                                               int fft_size, double frame_period, int fs, const int *y_lengths,
                                               int y_stride, int nbit, void *y) {
  if (!h || !f0 || !coded_spectral_envelope || !y || n_utts < 0 || fs <= 0 || frame_period <= 0)
    return WORLD_B200_EINVAL;
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  Ctx *ctx = ctx_of(h);
  if (nbit != 0 && nbit != 16) {
    ctx->last_error = "synthesis_coded_host: nbit must be 0 (double) or 16 (int16)";
    return WORLD_B200_EINVAL;
  }
  int lg = 0;
  int rc = synthesis_fft(ctx, fft_size, &lg);
  if (rc) return rc;
  CodedRows coded;
  rc = synthesis_coded_tables(ctx, fs, fft_size, number_of_dimensions, coded_aperiodicity != nullptr, &coded);
  if (rc) return rc;
  if (n_utts == 0) return 0;
  // every length is checked before the first chunk is queued
  std::vector<int> lens((size_t)2 * n_utts);
  rc = synthesis_lengths(ctx, f0_lengths, n_utts, f0_stride, y_lengths, y_stride, lens.data());
  if (rc) return rc;
  coded.sp = coded_spectral_envelope;
  coded.ap = coded.tap.dims > 0 ? coded_aperiodicity : nullptr;
  return synthesis_pipeline(h, &coded, lg, f0, f0_lengths, n_utts, f0_stride, fft_size, frame_period, fs, y_lengths,
                            y_stride, lens.data(), nbit, y);
}

extern "C" int world_b200_analyze_host(WorldB200 *h, const double *x, int n_utts, int x_stride,
                                       const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                       double *time_axis, double *f0, int f0_stride, double *spectrogram,
                                       double *aperiodicity) {
  if (!h || !x || !opt || n_utts < 0 || fs <= 0 || x_stride <= 0 || f0_stride <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  return analyze_pipeline(h, x, 0, n_utts, x_stride, x_lengths, fs, opt, nullptr, nullptr, 0, time_axis, f0, f0_stride,
                          spectrogram, aperiodicity);
}

// analyze_host with per-utterance options of one F0 method (harvest_options or dio_options)
static int analyze_host_per_utt(WorldB200 *h, const double *x, int n_utts, int x_stride, const int *x_lengths, int fs,
                                const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                const DioOption *dio_options, double *time_axis, double *f0, int f0_stride,
                                double *spectrogram, double *aperiodicity) {
  if (!h || !x || !opt || n_utts < 0 || fs <= 0 || x_stride <= 0 || f0_stride <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  const int rc = check_chain_f0_options(ctx_of(h), opt, harvest_options, dio_options, n_utts, fs, "analyze_host");
  if (rc) return rc;
  return analyze_pipeline(h, x, 0, n_utts, x_stride, x_lengths, fs, opt, harvest_options, dio_options, 0, time_axis, f0,
                          f0_stride, spectrogram, aperiodicity);
}

extern "C" int world_b200_analyze_host_options(WorldB200 *h, const double *x, int n_utts, int x_stride,
                                               const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                               const HarvestOption *harvest_options, double *time_axis, double *f0,
                                               int f0_stride, double *spectrogram, double *aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  return analyze_host_per_utt(h, x, n_utts, x_stride, x_lengths, fs, opt, harvest_options, nullptr, time_axis, f0,
                              f0_stride, spectrogram, aperiodicity);
}

extern "C" int world_b200_analyze_host_dio_options(WorldB200 *h, const double *x, int n_utts, int x_stride,
                                                   const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                   const DioOption *dio_options, double *time_axis, double *f0,
                                                   int f0_stride, double *spectrogram, double *aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  return analyze_host_per_utt(h, x, n_utts, x_stride, x_lengths, fs, opt, nullptr, dio_options, time_axis, f0,
                              f0_stride, spectrogram, aperiodicity);
}

// analyze_coded_host with per-utterance options of one F0 method, or none (both nullptr)
static int analyze_coded_host_impl(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths,
                                   int fs, const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options,
                                   const DioOption *dio_options, int number_of_dimensions, double *time_axis,
                                   double *f0, int f0_stride, double *coded_spectral_envelope,
                                   double *coded_aperiodicity) {
  if (!h || !x || !opt || n_utts < 0 || fs <= 0 || x_stride <= 0 || f0_stride <= 0) return WORLD_B200_EINVAL;
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  if (nbit != 0 && nbit != 8 && nbit != 16 && nbit != 24 && nbit != 32) return WORLD_B200_EINVAL;
  if (number_of_dimensions < 1 || number_of_dimensions > opt->cheaptrick.fft_size / 4 + 1) {
    ctx_of(h)->last_error = "analyze_coded_host: number_of_dimensions must be in [1, fft_size/4 + 1]";
    return WORLD_B200_EINVAL;
  }
  const int rc = check_chain_f0_options(ctx_of(h), opt, harvest_options, dio_options, n_utts, fs, "analyze_coded_host");
  if (rc) return rc;
  return analyze_pipeline(h, x, nbit, n_utts, x_stride, x_lengths, fs, opt, harvest_options, dio_options,
                          number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope, coded_aperiodicity);
}

extern "C" int world_b200_analyze_coded_host(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride,
                                             const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                             int number_of_dimensions, double *time_axis, double *f0, int f0_stride,
                                             double *coded_spectral_envelope, double *coded_aperiodicity) {
  return analyze_coded_host_impl(h, x, nbit, n_utts, x_stride, x_lengths, fs, opt, nullptr, nullptr,
                                 number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope,
                                 coded_aperiodicity);
}

extern "C" int world_b200_analyze_coded_host_options(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride,
                                                     const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                     const HarvestOption *harvest_options, int number_of_dimensions,
                                                     double *time_axis, double *f0, int f0_stride,
                                                     double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  return analyze_coded_host_impl(h, x, nbit, n_utts, x_stride, x_lengths, fs, opt, harvest_options, nullptr,
                                 number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope,
                                 coded_aperiodicity);
}

extern "C" int world_b200_analyze_coded_host_dio_options(WorldB200 *h, const void *x, int nbit, int n_utts,
                                                         int x_stride, const int *x_lengths, int fs,
                                                         const WorldB200AnalysisOption *opt,
                                                         const DioOption *dio_options, int number_of_dimensions,
                                                         double *time_axis, double *f0, int f0_stride,
                                                         double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  return analyze_coded_host_impl(h, x, nbit, n_utts, x_stride, x_lengths, fs, opt, nullptr, dio_options,
                                 number_of_dimensions, time_axis, f0, f0_stride, coded_spectral_envelope,
                                 coded_aperiodicity);
}

// ------------------------------------------------------------------ legacy single-utterance API
namespace {
std::mutex g_legacy_mutex;
WorldB200 *g_legacy = nullptr;

WorldB200 *legacy_ctx() {
  if (!g_legacy) {
    int dev = 0;
    if (const char *e = getenv("WORLD_B200_DEVICE")) dev = atoi(e);
    if (world_b200_create(dev, &g_legacy) != 0) {
      fprintf(stderr, "world_b200: cannot create a CUDA context for the legacy API (no CPU path)\n");
      g_legacy = nullptr;
    }
  }
  return g_legacy;
}

void report(WorldB200 *h, const char *fn, int rc) {
  if (rc) fprintf(stderr, "world_b200: %s failed (%d): %s\n", fn, rc, h ? world_b200_last_error(h) : "no CUDA context");
}

// The reference's void API cannot report an error: when a legacy call fails the caller's outputs are set to
// defined values (f0 / time axis 0 = "unvoiced", aperiodicity 1 - 1e-12 = the reference's default row,
// d4c.cpp:323-328, spectral envelope 1e-12, waveform 0) instead of being left uninitialised.
void fill(double *p, size_t n, double v) {
  if (p) for (size_t i = 0; i < n; ++i) p[i] = v;
}
void fill_rows(double **rows, int n_rows, int width, double v) {
  if (rows) for (int i = 0; i < n_rows; ++i) fill(rows[i], (size_t)width, v);
}

// stage(x dev, t dev, f0 dev) helpers share the upload of x / time / f0
struct Legacy1 {
  WorldB200 *h; Ctx *ctx;
  double *x = nullptr, *t = nullptr, *f = nullptr;
  int rc = 0;
  std::unique_ptr<DeviceGuard> guard;   // the legacy context's device is current while this object lives
  Legacy1(const double *xh, int x_length, const double *th, const double *fh, int f0_length) {
    h = legacy_ctx();
    ctx = h ? ctx_of(h) : nullptr;
    if (!h) { rc = WORLD_B200_ECUDA; return; }
    guard.reset(new DeviceGuard(ctx));
    x = (double *)dev_malloc(ctx, (size_t)x_length * 8);
    t = (double *)dev_malloc(ctx, (size_t)imax(1, f0_length) * 8);
    f = (double *)dev_malloc(ctx, (size_t)imax(1, f0_length) * 8);
    if (!x || !t || !f) { rc = WORLD_B200_ENOMEM; return; }
    rc = dev_memcpy_h2d(ctx, x, xh, (size_t)x_length * 8);
    if (!rc && th) rc = dev_memcpy_h2d(ctx, t, th, (size_t)f0_length * 8);
    if (!rc && fh) rc = dev_memcpy_h2d(ctx, f, fh, (size_t)f0_length * 8);
    if (!rc && !th) rc = dev_memset(ctx, t, 0, (size_t)imax(1, f0_length) * 8);
    if (!rc && !fh) rc = dev_memset(ctx, f, 0, (size_t)imax(1, f0_length) * 8);
  }
  ~Legacy1() { dev_free(x); dev_free(t); dev_free(f); }
};
}  // namespace

extern "C" {

void Dio(const double *x, int x_length, int fs, const DioOption *option, double *temporal_positions, double *f0) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  const int L = GetSamplesForDIO(fs, x_length, option->frame_period);
  Legacy1 d(x, x_length, nullptr, nullptr, L);
  int rc = d.rc;
  if (!rc) rc = world_b200_dio_batch(d.h, d.x, 1, x_length, nullptr, fs, option, d.t, d.f, L);
  if (!rc) rc = dev_memcpy_d2h(d.ctx, temporal_positions, d.t, (size_t)L * 8);
  if (!rc) rc = dev_memcpy_d2h(d.ctx, f0, d.f, (size_t)L * 8);
  if (!rc) rc = world_b200_synchronize(d.h);
  if (rc) { fill(temporal_positions, (size_t)L, 0.0); fill(f0, (size_t)L, 0.0); }
  report(d.h, "Dio", rc);
}

void Harvest(const double *x, int x_length, int fs, const HarvestOption *option, double *temporal_positions,
             double *f0) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  const int L = GetSamplesForHarvest(fs, x_length, option->frame_period);
  Legacy1 d(x, x_length, nullptr, nullptr, L);
  int rc = d.rc;
  if (!rc) rc = world_b200_harvest_batch(d.h, d.x, 1, x_length, nullptr, fs, option, d.t, d.f, L);
  if (!rc) rc = dev_memcpy_d2h(d.ctx, temporal_positions, d.t, (size_t)L * 8);
  if (!rc) rc = dev_memcpy_d2h(d.ctx, f0, d.f, (size_t)L * 8);
  if (!rc) rc = world_b200_synchronize(d.h);
  if (rc) { fill(temporal_positions, (size_t)L, 0.0); fill(f0, (size_t)L, 0.0); }
  report(d.h, "Harvest", rc);
}

void StoneMask(const double *x, int x_length, int fs, const double *temporal_positions, const double *f0,
               int f0_length, double *refined_f0) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  Legacy1 d(x, x_length, temporal_positions, f0, f0_length);
  int rc = d.rc;
  if (!rc) rc = world_b200_stonemask_batch(d.h, d.x, 1, x_length, nullptr, fs, d.t, d.f, nullptr, f0_length, d.f);
  if (!rc) rc = dev_memcpy_d2h(d.ctx, refined_f0, d.f, (size_t)f0_length * 8);
  if (!rc) rc = world_b200_synchronize(d.h);
  if (rc) fill(refined_f0, (size_t)f0_length, 0.0);
  report(d.h, "StoneMask", rc);
}

static void rows_out(Legacy1 &d, const char *name, int rc, double *dev_rows, int f0_length, int bins, double **rows,
                     double fail_value) {
  std::vector<double> flat((size_t)f0_length * bins);
  if (!rc) rc = dev_memcpy_d2h(d.ctx, flat.data(), dev_rows, flat.size() * 8);
  if (!rc) rc = world_b200_synchronize(d.h);
  if (!rc)
    for (int i = 0; i < f0_length; ++i) memcpy(rows[i], flat.data() + (size_t)i * bins, (size_t)bins * 8);
  else
    fill_rows(rows, f0_length, bins, fail_value);
  report(d.h, name, rc);
}

void CheapTrick(const double *x, int x_length, int fs, const double *temporal_positions, const double *f0,
                int f0_length, const CheapTrickOption *option, double **spectrogram) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  Legacy1 d(x, x_length, temporal_positions, f0, f0_length);
  const int bins = option->fft_size / 2 + 1;
  double *rows = d.rc ? nullptr : (double *)dev_malloc(d.ctx, (size_t)imax(1, f0_length) * bins * 8);
  int rc = d.rc ? d.rc : (rows ? 0 : WORLD_B200_ENOMEM);
  if (!rc) rc = world_b200_cheaptrick_batch(d.h, d.x, 1, x_length, nullptr, fs, d.t, d.f, nullptr, f0_length, option, rows);
  rows_out(d, "CheapTrick", rc, rows, f0_length, bins, spectrogram, kTiny);
  dev_free(rows);
}

void D4C(const double *x, int x_length, int fs, const double *temporal_positions, const double *f0, int f0_length,
         int fft_size, const D4COption *option, double **aperiodicity) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  Legacy1 d(x, x_length, temporal_positions, f0, f0_length);
  const int bins = fft_size / 2 + 1;
  double *rows = d.rc ? nullptr : (double *)dev_malloc(d.ctx, (size_t)imax(1, f0_length) * bins * 8);
  int rc = d.rc ? d.rc : (rows ? 0 : WORLD_B200_ENOMEM);
  if (!rc) rc = world_b200_d4c_batch(d.h, d.x, 1, x_length, nullptr, fs, d.t, d.f, nullptr, f0_length, fft_size, option, rows);
  rows_out(d, "D4C", rc, rows, f0_length, bins, aperiodicity, 1.0 - kTiny);
  dev_free(rows);
}

void Synthesis(const double *f0, int f0_length, const double *const *spectrogram, const double *const *aperiodicity,
               int fft_size, double frame_period, int fs, int y_length, double *y) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  WorldB200 *h = legacy_ctx();
  if (!h) { fill(y, (size_t)imax(0, y_length), 0.0); report(h, "Synthesis", WORLD_B200_ECUDA); return; }
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  Ctx *ctx = ctx_of(h);
  const int bins = fft_size / 2 + 1;
  std::vector<double> flat((size_t)f0_length * bins);
  double *d_f0 = (double *)dev_malloc(ctx, (size_t)f0_length * 8);
  double *d_sp = (double *)dev_malloc(ctx, flat.size() * 8), *d_ap = (double *)dev_malloc(ctx, flat.size() * 8);
  double *d_y = (double *)dev_malloc(ctx, (size_t)y_length * 8);
  int rc = (d_f0 && d_sp && d_ap && d_y) ? 0 : WORLD_B200_ENOMEM;
  if (!rc) rc = dev_memcpy_h2d(ctx, d_f0, f0, (size_t)f0_length * 8);
  for (int pass = 0; pass < 2 && !rc; ++pass) {
    const double *const *rows = pass == 0 ? spectrogram : aperiodicity;
    for (int i = 0; i < f0_length; ++i) memcpy(flat.data() + (size_t)i * bins, rows[i], (size_t)bins * 8);
    rc = dev_memcpy_h2d(ctx, pass == 0 ? d_sp : d_ap, flat.data(), flat.size() * 8);
    if (!rc) rc = dev_sync(ctx);  // flat is reused
  }
  if (!rc) rc = world_b200_synthesis_batch(h, d_f0, nullptr, 1, f0_length, d_sp, d_ap, fft_size, frame_period, fs,
                                           nullptr, y_length, d_y);
  if (!rc) rc = dev_memcpy_d2h(ctx, y, d_y, (size_t)y_length * 8);
  if (!rc) rc = world_b200_synchronize(h);
  if (rc) fill(y, (size_t)imax(0, y_length), 0.0);
  report(h, "Synthesis", rc);
  dev_free(d_f0); dev_free(d_sp); dev_free(d_ap); dev_free(d_y);
}

// ---- codec.h: rows in, rows out, one utterance
static void codec_rows(const char *name, const double *const *in_rows, int f0_length, int in_w, int out_w,
                       double **out_rows, int (*run)(WorldB200 *, const double *, double *, void *), void *arg) {
  std::lock_guard<std::mutex> lock(g_legacy_mutex);
  WorldB200 *h = legacy_ctx();
  if (f0_length <= 0 || out_w <= 0) return;
  if (!h) { fill_rows(out_rows, f0_length, out_w, 0.0); report(h, name, WORLD_B200_ECUDA); return; }
  DeviceGuard guard_(reinterpret_cast<const Ctx *>(h));  // Ctx is the first member of WorldB200
  Ctx *ctx = ctx_of(h);
  std::vector<double> flat_in((size_t)f0_length * imax(1, in_w)), flat_out((size_t)f0_length * out_w);
  for (int i = 0; i < f0_length && in_w > 0; ++i) memcpy(flat_in.data() + (size_t)i * in_w, in_rows[i], (size_t)in_w * 8);
  double *d_in = (double *)dev_malloc(ctx, flat_in.size() * 8), *d_out = (double *)dev_malloc(ctx, flat_out.size() * 8);
  int rc = (d_in && d_out) ? 0 : WORLD_B200_ENOMEM;
  if (!rc) rc = dev_memcpy_h2d(ctx, d_in, flat_in.data(), flat_in.size() * 8);
  if (!rc) rc = run(h, d_in, d_out, arg);
  if (!rc) rc = dev_memcpy_d2h(ctx, flat_out.data(), d_out, flat_out.size() * 8);
  if (!rc) rc = world_b200_synchronize(h);
  if (!rc)
    for (int i = 0; i < f0_length; ++i) memcpy(out_rows[i], flat_out.data() + (size_t)i * out_w, (size_t)out_w * 8);
  else
    fill_rows(out_rows, f0_length, out_w, 0.0);
  report(h, name, rc);
  dev_free(d_in); dev_free(d_out);
}

struct CodecArgs { int f0_length, fs, fft_size, dims; };

void CodeAperiodicity(const double *const *aperiodicity, int f0_length, int fs, int fft_size,
                      double **coded_aperiodicity) {
  CodecArgs a = {f0_length, fs, fft_size, 0};
  codec_rows("CodeAperiodicity", aperiodicity, f0_length, fft_size / 2 + 1, GetNumberOfAperiodicities(fs),
             coded_aperiodicity, [](WorldB200 *h, const double *in, double *out, void *p) {
               const CodecArgs *a = (const CodecArgs *)p;
               return world_b200_code_aperiodicity_batch(h, in, 1, nullptr, a->f0_length, a->fs, a->fft_size, out);
             }, &a);
}

void DecodeAperiodicity(const double *const *coded_aperiodicity, int f0_length, int fs, int fft_size,
                        double **aperiodicity) {
  CodecArgs a = {f0_length, fs, fft_size, 0};
  codec_rows("DecodeAperiodicity", coded_aperiodicity, f0_length, GetNumberOfAperiodicities(fs), fft_size / 2 + 1,
             aperiodicity, [](WorldB200 *h, const double *in, double *out, void *p) {
               const CodecArgs *a = (const CodecArgs *)p;
               return world_b200_decode_aperiodicity_batch(h, in, 1, nullptr, a->f0_length, a->fs, a->fft_size, out);
             }, &a);
}

void CodeSpectralEnvelope(const double *const *spectrogram, int f0_length, int fs, int fft_size,
                          int number_of_dimensions, double **coded_spectral_envelope) {
  CodecArgs a = {f0_length, fs, fft_size, number_of_dimensions};
  codec_rows("CodeSpectralEnvelope", spectrogram, f0_length, fft_size / 2 + 1, number_of_dimensions,
             coded_spectral_envelope, [](WorldB200 *h, const double *in, double *out, void *p) {
               const CodecArgs *a = (const CodecArgs *)p;
               return world_b200_code_spectral_envelope_batch(h, in, 1, nullptr, a->f0_length, a->fs, a->fft_size,
                                                              a->dims, out);
             }, &a);
}

void DecodeSpectralEnvelope(const double *const *coded_spectral_envelope, int f0_length, int fs, int fft_size,
                            int number_of_dimensions, double **spectrogram) {
  CodecArgs a = {f0_length, fs, fft_size, number_of_dimensions};
  codec_rows("DecodeSpectralEnvelope", coded_spectral_envelope, f0_length, number_of_dimensions, fft_size / 2 + 1,
             spectrogram, [](WorldB200 *h, const double *in, double *out, void *p) {
               const CodecArgs *a = (const CodecArgs *)p;
               return world_b200_decode_spectral_envelope_batch(h, in, 1, nullptr, a->f0_length, a->fs, a->fft_size,
                                                                a->dims, out);
             }, &a);
}

}  // extern "C"
