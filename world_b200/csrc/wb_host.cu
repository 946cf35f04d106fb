// wb_host.cu -- host-pointer entry points built on the device-pointer ABI:
//   * world_b200_analyze_host(): {Dio+StoneMask | Harvest} -> CheapTrick -> D4C for N host
//     waveforms, upload / compute / download pipelined over utterance chunks on three streams;
//   * world_b200_synthesis_coded_host(): the way back, f0 + coded rows -> waveforms or 16-bit PCM,
//     pipelined the same way;
//   * the reference's own single-utterance functions (Dio, Harvest, StoneMask, CheapTrick, D4C;
//     src/world/*.h) as n_utts = 1 batches on a lazily created process-wide context, so existing
//     callers relink unchanged.  They keep the reference's `void` signature; failures are
//     reported on stderr and leave the outputs zero-filled.
#include "wb_chain.h"
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <memory>
#include <mutex>
#include <chrono>
#include <algorithm>
#include <string.h>

using namespace wb;

namespace {

// The scaffold of the host pipelines: uploads on s_in, kernels on the context's stream, downloads on s_out, the events
// that order buffer reuse between the three, the pipeline's pooled device buffers and the WB_HOST_TRACE timeline.  On
// the host emulation the copies are memcpy and the stream operations do nothing.
//
// Ordering rules.  open() makes s_in wait for the work already on the context's stream.  finish() synchronises s_in, the
// context's stream and s_out, in that order, and only then releases the buffers; the destructor does the same on any
// return path that did not reach finish(), so no buffer goes back to the pool while a copy may still use it.
class HostPipe {
 public:
  enum Stream { IN, RUN, OUT };

  HostPipe(WorldB200 *h, const char *who)
      : ctx_(&h->c), who_(who), trace_(getenv("WB_HOST_TRACE") != nullptr), t0_(std::chrono::steady_clock::now()) {}
  HostPipe(const HostPipe &) = delete;
  HostPipe &operator=(const HostPipe &) = delete;
  ~HostPipe() { close(); }

  // the two streams and n_events events (indices 0 .. n_events - 1); ECUDA with last_error when one cannot be made
  int open(int n_events) {
#ifndef WB_EMU
    if (cudaStreamCreateWithFlags(&s_in_, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&s_out_, cudaStreamNonBlocking) != cudaSuccess)
      return fail("cudaStreamCreate failed");
    for (int i = 0; i <= n_events; ++i) {
      cudaEvent_t e;
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return fail("cudaEventCreate failed");
      ev_.push_back(e);
    }
    mark("start", 0, RUN);
    // the uploads start after the work already on the context's stream: a pooled buffer released by a stream-ordered
    // call (the PCM buffer of world_b200_analyze_coded_batch) may still be read there
    cudaEventRecord(ev_[n_events], ctx_->stream);
    cudaStreamWaitEvent(s_in_, ev_[n_events], 0);
#else
    (void)n_events;
#endif
    return 0;
  }

  // a pooled device buffer of `bytes` (none for 0), released by the scaffold; ENOMEM with last_error when none is left
  template <class T>
  int buffer(size_t bytes, T **p) {
    *p = bytes ? (T *)pool_acquire(ctx_, bytes) : nullptr;
    if (*p) bufs_.push_back(*p);
    return *p || !bytes ? 0 : WORLD_B200_ENOMEM;
  }

  void h2d(void *dst, const void *src, size_t bytes) {
#ifndef WB_EMU
    cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s_in_);
#else
    memcpy(dst, src, bytes);
#endif
  }
  void d2h(void *dst, const void *src, size_t bytes) {
#ifndef WB_EMU
    cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s_out_);
#else
    memcpy(dst, src, bytes);
#endif
  }
  void record(int ev, Stream s) {
#ifndef WB_EMU
    cudaEventRecord(ev_[ev], stream(s));
#else
    (void)ev; (void)s;
#endif
  }
  void wait(Stream s, int ev) {
#ifndef WB_EMU
    cudaStreamWaitEvent(stream(s), ev_[ev], 0);
#else
    (void)s; (void)ev;
#endif
  }
  // WB_HOST_TRACE=1: timeline of this call on stderr (timing events on the three streams + host clock)
  void mark(const char *what, int idx, Stream s) {
#ifndef WB_EMU
    if (!trace_) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, stream(s));
    marks_.push_back(Mark{what, idx, ms(), e});
#else
    (void)what; (void)idx; (void)s;
#endif
  }

  // Waits for the three streams, turns a sticky error into "<who> pipeline: ...", prints the trace (its first line is
  // "[wb trace] <header>: all work issued at ...") and releases the streams, events and buffers.
  int finish(int rc, const char *header) {
    const double issued_ms = ms();
#ifndef WB_EMU
    // copies and memsets above are not checked one by one: a failure is sticky and surfaces here
    cudaError_t e = cudaStreamSynchronize(s_in_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx_->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s_out_);
    synced_ = true;
    if (e != cudaSuccess && !rc) {
      ctx_->last_error = std::string(who_) + " pipeline: " + cudaGetErrorString(e);
      rc = WORLD_B200_ECUDA;
    }
#endif
    if (trace_) {
      fprintf(stderr, "[wb trace] %s: all work issued at %.1f ms, finished at %.1f ms (host clock)\n", header, issued_ms,
              ms());
#ifndef WB_EMU
      for (size_t i = 1; i < marks_.size(); ++i) {
        float gpu_ms = 0.f;
        cudaEventElapsedTime(&gpu_ms, marks_[0].ev, marks_[i].ev);
        fprintf(stderr, "[wb trace] %-9s %3d  issued %8.1f  gpu %8.1f\n", marks_[i].what, marks_[i].idx, marks_[i].host_ms,
                gpu_ms);
      }
#endif
    }
    close();
#ifndef WB_EMU
    if (!rc) {
      const cudaError_t last = cudaGetLastError();
      if (last != cudaSuccess) { ctx_->last_error = cudaGetErrorString(last); rc = WORLD_B200_ECUDA; }
    }
#endif
    return rc;
  }

 private:
  double ms() const {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0_).count();
  }
#ifndef WB_EMU
  struct Mark { const char *what; int idx; double host_ms; cudaEvent_t ev; };
  cudaStream_t stream(Stream s) const { return s == IN ? s_in_ : s == OUT ? s_out_ : ctx_->stream; }
  int fail(const char *what) {
    ctx_->last_error = what;
    cudaGetLastError();
    return WORLD_B200_ECUDA;
  }
#endif
  void close() {
#ifndef WB_EMU
    if (!synced_) {
      if (s_in_) cudaStreamSynchronize(s_in_);
      cudaStreamSynchronize(ctx_->stream);
      if (s_out_) cudaStreamSynchronize(s_out_);
      synced_ = true;
    }
    for (auto &m : marks_) cudaEventDestroy(m.ev);
    for (cudaEvent_t e : ev_) cudaEventDestroy(e);
    if (s_in_) cudaStreamDestroy(s_in_);
    if (s_out_) cudaStreamDestroy(s_out_);
    marks_.clear(); ev_.clear(); s_in_ = s_out_ = nullptr;
#endif
    for (void *p : bufs_) pool_release(ctx_, p);
    bufs_.clear();
  }

  Ctx *ctx_;
  const char *who_;
  const bool trace_;
  const std::chrono::steady_clock::time_point t0_;
  std::vector<void *> bufs_;
#ifndef WB_EMU
  cudaStream_t s_in_ = nullptr, s_out_ = nullptr;
  std::vector<cudaEvent_t> ev_;   // the pipeline's events, then the start event
  std::vector<Mark> marks_;
  bool synced_ = false;
#endif
};

// One pipeline for both host entry points.  nbit == 0: x holds doubles; otherwise little-endian PCM that
// is widened on the device (row f3).  dims == 0: the full spectrogram / aperiodicity rows go back to the
// host; dims > 0: they stay on the device and only their coded rows (row f2), written by the fused frame kernels
// (world_b200_cheaptrick_coded_batch / world_b200_d4c_coded_batch), are downloaded.
//
// Two granularities.  The F0 stage runs on OUTER chunks (default 512 utterances): its per-utterance
// kernels (contour tracking, smoothing, decimation) are latency bound -- one launch costs the same
// for 96 or 500 utterances -- so few large launches beat many small ones.  CheapTrick / D4C run
// on SUB-chunks (default 128 utterances) whose rows start their trip over PCIe as soon as they exist: the
// un-overlapped tail is one sub-chunk.  Result buffers form a ring two outer chunks deep, so downloads
// may lag behind the frame kernels and catch up under the next outer chunk's F0 stage.  Streams and events: HostPipe.
// The whole request is checked (chain_plan) before the first upload; the per-utterance option arrays are split with the
// outer chunks.  time_axis and f0 may be NULL: they are computed on the device and not downloaded.
int analyze_pipeline(WorldB200 *h, const ChainRequest &r) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  const char *who = r.coded ? "analyze_coded_host" : "analyze_host";
  if (r.f0_stride <= 0) {
    ctx->last_error = std::string(who) + ": f0_stride must be > 0";
    return WORLD_B200_EINVAL;
  }
  ChainPlan plan;
  int rc = chain_plan(ctx, r, who, &plan);
  if (rc || r.n == 0) return rc;
  const int n_utts = r.n, nbit = r.nbit, x_stride = r.x_stride, f0_stride = r.f0_stride;
  const size_t in_bytes = nbit ? (size_t)(nbit / 8) : 8;
  const size_t sp_row = plan.sp_row, ap_row = plan.ap_row;
  const bool want_sp = plan.want_sp, want_ap = plan.want_ap;
  const StagePlan &sizes = want_sp ? plan.ct : plan.d4;   // each utterance's fft_size (D4C runs at CheapTrick's)
  double *time_axis = r.time_axis, *f0 = r.f0, *out_sp = r.spectrogram, *out_ap = r.aperiodicity;

  int sub = 128, outer = 512;
  if (const char *e = getenv("WB_HOST_SUB")) sub = atoi(e) > 0 ? atoi(e) : sub;
  if (const char *e = getenv("WB_HOST_CHUNK")) outer = atoi(e) > 0 ? atoi(e) : outer;
  sub = imin(sub, n_utts);
  // a third of the scratch budget for this pipeline's own buffers: two outer sets + the result ring
  const size_t third = ctx->scratch_budget / 3;
  const size_t per_outer = (size_t)x_stride * (in_bytes + (nbit ? 8 : 0)) + (size_t)f0_stride * 16;
  const size_t per_sub_out = (size_t)f0_stride * ((want_sp ? sp_row : 0) + (want_ap ? ap_row : 0)) * 8;
  outer = imin(outer, (int)dmax((double)sub, (double)(third / 3) / (double)(2 * per_outer)));
  outer = imax(sub, outer / sub * sub);
  outer = imin(outer, (n_utts + sub - 1) / sub * sub);
  const int subs_per_outer = outer / sub;
  const double ring_budget = (double)third - (double)imin(n_utts, outer) * 2.0 * (double)per_outer;
  int ring = 2 * subs_per_outer;
  if (per_sub_out > 0)
    ring = imax(2, imin(ring, (int)dmax(0.0, ring_budget / ((double)sub * (double)per_sub_out))));
  ring = imin(ring, (n_utts + sub - 1) / sub);
  if (ring < 1) ring = 1;

  // events: two of each per outer buffer set, then a "computed" and a "downloaded" event per result slot
  enum { EV_IN = 0, EV_CDONE = 2, EV_F0 = 4, EV_TF = 6, EV_SUB_DONE = 8 };
  const int ev_sub_out = EV_SUB_DONE + ring;
  HostPipe p(h, "analyze");
  rc = p.open(EV_SUB_DONE + 2 * ring);
  if (rc) return rc;
  unsigned char *din[2] = {nullptr, nullptr};
  double *dx[2] = {nullptr, nullptr}, *dt[2] = {nullptr, nullptr}, *df[2] = {nullptr, nullptr};
  std::vector<double *> dsp(ring, nullptr), dap(ring, nullptr);   // the result ring: full or coded rows
  const int n_outer_bufs = n_utts > outer ? 2 : 1;
  for (int i = 0; i < n_outer_bufs && !rc; ++i) {
    rc = p.buffer((size_t)outer * x_stride * in_bytes, &din[i]);
    if (!rc && nbit) rc = p.buffer((size_t)outer * x_stride * 8, &dx[i]);
    if (!rc) rc = p.buffer((size_t)outer * f0_stride * 8, &dt[i]);
    if (!rc) rc = p.buffer((size_t)outer * f0_stride * 8, &df[i]);
  }
  for (int i = 0; i < ring && !rc; ++i) {
    if (want_sp) rc = p.buffer((size_t)sub * f0_stride * sp_row * 8, &dsp[i]);
    if (!rc && want_ap) rc = p.buffer((size_t)sub * f0_stride * ap_row * 8, &dap[i]);
  }
  int it = 0, g = 0;   // outer chunk counter, global sub-chunk counter
  for (int u0 = 0; u0 < n_utts && !rc; u0 += outer, ++it) {
    const int n = imin(outer, n_utts - u0);
    const int s = it & 1;
    const int *fl = plan.f_len.data() + u0;
    const size_t fsz = (size_t)n * f0_stride;
    if (it >= 2) p.wait(HostPipe::IN, EV_CDONE + s);   // kernels of outer chunk it-2 read din[s] / dx[s]
    p.h2d(din[s], (const unsigned char *)r.x + (size_t)u0 * x_stride * in_bytes, (size_t)n * x_stride * in_bytes);
    p.record(EV_IN + s, HostPipe::IN);
    p.mark("h2d_done", it, HostPipe::IN);
    p.wait(HostPipe::RUN, EV_IN + s);
    if (it >= 2) p.wait(HostPipe::RUN, EV_TF + s);   // time_axis / f0 of it-2 are on the host
    p.mark("f0_begin", it, HostPipe::RUN);
    if (nbit)
      rc = world_b200_pcm_to_double_batch(h, din[s], nbit, n, x_stride, r.x_lengths ? r.x_lengths + u0 : nullptr, dx[s]);
    if (rc) break;
    dev_memset(ctx, dt[s], 0, fsz * 8);
    dev_memset(ctx, df[s], 0, fsz * 8);
    const double *xd = nbit ? dx[s] : (const double *)din[s];
    rc = chain_f0(h, r, plan, u0, n, xd, dt[s], df[s]);
    if (rc) break;
    p.record(EV_F0 + s, HostPipe::RUN);
    p.mark("f0_end", it, HostPipe::RUN);
    p.wait(HostPipe::OUT, EV_F0 + s);
    if (time_axis) p.d2h(time_axis + (size_t)u0 * f0_stride, dt[s], fsz * 8);
    if (f0) p.d2h(f0 + (size_t)u0 * f0_stride, df[s], fsz * 8);
    p.record(EV_TF + s, HostPipe::OUT);
    // Sub-chunk size.  A sub-chunk's rows go to the host while the next one is computed, and in the full-row mode a
    // sub-chunk takes ~12 % longer to download than to compute: after the LAST outer chunk the copy engine is the
    // critical path, finishing (first sub-chunk's compute + every download) after the chunk's Harvest -- ~50 ms behind
    // the kernels of a 850 ms step at 1024 x 10 s with sub-chunks of 128.  Quarter-size sub-chunks there start the
    // downloads earlier and leave a shorter last one (~25 ms behind).
    const bool taper = !r.coded && u0 + outer >= n_utts;
    int taper_min = 16;   // (WB_HOST_TAPER_MIN: tests exercise the path with a handful of utterances)
    if (const char *e = getenv("WB_HOST_TAPER_MIN")) taper_min = imax(1, atoi(e));
    const int sub_here = taper ? imax(imin(sub, taper_min), sub / 4) : sub;
    for (int v0 = 0; v0 < n && !rc && (want_sp || want_ap); v0 += sub_here, ++g) {
      const int m = imin(sub_here, n - v0);
      const int slot = g % ring;
      const int *sfl = fl + v0;
      const size_t ssz = (size_t)m * f0_stride;
      const double *sx = xd + (size_t)v0 * x_stride, *st = dt[s] + (size_t)v0 * f0_stride, *sf = df[s] + (size_t)v0 * f0_stride;
      if (g >= ring) p.wait(HostPipe::RUN, ev_sub_out + slot);   // the slot's previous rows are on the host
      // whole padded rows are downloaded: frames beyond an utterance's length, and full-row values beyond its
      // fft_size / 2 + 1 (per-utterance sizes, or a wider row_stride), read as zero on the host
      bool ragged = false;
      for (int i = 0; i < m; ++i)
        ragged = ragged || sfl[i] != f0_stride || (!r.coded && (size_t)(sizes.fft_size[u0 + v0 + i] / 2 + 1) != sp_row);
      if (ragged) {
        if (want_sp) dev_memset(ctx, dsp[slot], 0, ssz * sp_row * 8);
        if (want_ap) dev_memset(ctx, dap[slot], 0, ssz * ap_row * 8);
      }
      rc = chain_spectral(h, r, plan, u0 + v0, m, sx, st, sf, want_sp ? dsp[slot] : nullptr,
                          want_ap ? dap[slot] : nullptr);
      if (rc) break;
      const size_t row0 = (size_t)(u0 + v0) * f0_stride;
      p.record(EV_SUB_DONE + slot, HostPipe::RUN);
      p.mark("sub_end", g, HostPipe::RUN);
      p.wait(HostPipe::OUT, EV_SUB_DONE + slot);
      if (want_sp) p.d2h(out_sp + row0 * sp_row, dsp[slot], ssz * sp_row * 8);
      if (want_ap) p.d2h(out_ap + row0 * ap_row, dap[slot], ssz * ap_row * 8);
      p.record(ev_sub_out + slot, HostPipe::OUT);
      p.mark("d2h_end", g, HostPipe::OUT);
    }
    p.record(EV_CDONE + s, HostPipe::RUN);
  }
  char header[96];
  snprintf(header, sizeof header, "outer %d sub %d ring %d n %d", outer, sub, ring, n_utts);
  rc = p.finish(rc, header);
  if (!rc) rc = world_b200_synchronize(h);
  return rc;
}

// The packed chains for host arrays.  Utterances go in chunks (at most WB_HOST_CHUNK, default 512, and as many as keep
// one chunk's device rows within a twelfth of the scratch budget: two input buffers and two output sets take a third).
// A chunk's samples [x_offsets[c0], x_offsets[c1]) go up as one copy on s_in, packed_run analyses them on the context's
// stream with chunk-relative offsets, and each output array's frames [f_off[c0], f_off[c1]) come back as one copy on
// s_out, so the upload of the next chunk and the download of the last overlap this chunk's kernels.  Full rows are
// zeroed first where an utterance is narrower than the row.  time_axis and f0 may be NULL: not downloaded.
int analyze_packed_pipeline(WorldB200 *h, const ChainRequest &r, long long *f_offsets) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
  ChainPlan plan;
  int rc = chain_plan(ctx, r, r.coded ? "analyze_coded_host_packed" : "analyze_host_packed", &plan);
  if (rc) return rc;
  if (f_offsets) std::copy(plan.f_off.begin(), plan.f_off.end(), f_offsets);
  const int n_utts = r.n;
  if (n_utts == 0) return 0;
  const long long *xo = r.x_offsets, *fo = plan.f_off.data();
  const size_t in_bytes = r.nbit ? (size_t)(r.nbit / 8) : 8;
  const bool want_sp = plan.want_sp, want_ap = plan.want_ap;
  const size_t sp_row = want_sp ? plan.sp_row : 0, ap_row = want_ap ? plan.ap_row : 0;
  const StagePlan &sizes = want_sp ? plan.ct : plan.d4;   // each utterance's fft_size (D4C runs at CheapTrick's)
  const size_t per_frame = (2 + sp_row + ap_row) * 8;
  int outer = 512;
  if (const char *e = getenv("WB_HOST_CHUNK")) outer = atoi(e) > 0 ? atoi(e) : outer;
  const size_t cap = ctx->scratch_budget / 12;
  auto bytes = [&](int c0, int c1) {
    return (size_t)(xo[c1] - xo[c0]) * in_bytes + (size_t)(fo[c1] - fo[c0]) * per_frame;
  };
  std::vector<int> bounds{0};
  while (bounds.back() < n_utts) {
    const int c0 = bounds.back();
    int c1 = c0 + 1;
    while (c1 < n_utts && c1 - c0 < outer && bytes(c0, c1 + 1) <= cap) ++c1;
    bounds.push_back(c1);
  }
  const int n_chunks = (int)bounds.size() - 1;
  size_t most_in = 0, most_frames = 0;
  for (int k = 0; k < n_chunks; ++k) {
    most_in = std::max(most_in, (size_t)(xo[bounds[k + 1]] - xo[bounds[k]]) * in_bytes);
    most_frames = std::max(most_frames, (size_t)(fo[bounds[k + 1]] - fo[bounds[k]]));
  }

  enum { EV_IN = 0, EV_CDONE = 2, EV_OUT = 4 };   // per buffer set: uploaded, computed, downloaded
  HostPipe p(h, "analyze_packed");
  rc = p.open(6);
  if (rc) return rc;
  unsigned char *din[2] = {nullptr, nullptr};
  double *dt[2] = {nullptr, nullptr}, *df[2] = {nullptr, nullptr}, *dsp[2] = {nullptr, nullptr},
         *dap[2] = {nullptr, nullptr};
  for (int i = 0; i < (n_chunks > 1 ? 2 : 1) && !rc; ++i) {
    rc = p.buffer(most_in, &din[i]);
    if (!rc) rc = p.buffer(most_frames * 8, &dt[i]);
    if (!rc) rc = p.buffer(most_frames * 8, &df[i]);
    if (!rc) rc = p.buffer(most_frames * sp_row * 8, &dsp[i]);
    if (!rc) rc = p.buffer(most_frames * ap_row * 8, &dap[i]);
  }
  for (int k = 0; k < n_chunks && !rc; ++k) {
    const int c0 = bounds[k], c1 = bounds[k + 1], s = k & 1;
    const size_t frames = (size_t)(fo[c1] - fo[c0]);
    if (k >= 2) p.wait(HostPipe::IN, EV_CDONE + s);   // the kernels of chunk k - 2 have read din[s]
    p.h2d(din[s], (const unsigned char *)r.x + (size_t)xo[c0] * in_bytes, (size_t)(xo[c1] - xo[c0]) * in_bytes);
    p.record(EV_IN + s, HostPipe::IN);
    p.mark("h2d_done", k, HostPipe::IN);
    p.wait(HostPipe::RUN, EV_IN + s);
    if (k >= 2) p.wait(HostPipe::RUN, EV_OUT + s);   // the rows of chunk k - 2 are on the host
    p.mark("run_begin", k, HostPipe::RUN);
    bool narrow = false;
    for (int u = c0; u < c1 && !r.coded; ++u) narrow = narrow || (size_t)(sizes.fft_size[u] / 2 + 1) != plan.sp_row;
    if (narrow && want_sp) rc = dev_memset(ctx, dsp[s], 0, frames * sp_row * 8);
    if (narrow && want_ap && !rc) rc = dev_memset(ctx, dap[s], 0, frames * ap_row * 8);
    if (!rc) rc = packed_run(h, r, plan, c0, c1, din[s], dt[s], df[s], dsp[s], dap[s]);
    if (rc) break;
    p.record(EV_CDONE + s, HostPipe::RUN);
    p.mark("run_end", k, HostPipe::RUN);
    p.wait(HostPipe::OUT, EV_CDONE + s);
    if (r.time_axis) p.d2h(r.time_axis + fo[c0], dt[s], frames * 8);
    if (r.f0) p.d2h(r.f0 + fo[c0], df[s], frames * 8);
    if (want_sp) p.d2h(r.spectrogram + (size_t)fo[c0] * sp_row, dsp[s], frames * sp_row * 8);
    if (want_ap) p.d2h(r.aperiodicity + (size_t)fo[c0] * ap_row, dap[s], frames * ap_row * 8);
    p.record(EV_OUT + s, HostPipe::OUT);
    p.mark("d2h_end", k, HostPipe::OUT);
  }
  char header[96];
  snprintf(header, sizeof header, "chunks %d n %d", n_chunks, n_utts);
  rc = p.finish(rc, header);
  if (!rc) rc = world_b200_synchronize(h);
  return rc;
}

// The chunk loop of the synthesis and transform pipelines.  Chunk k is utterances [bounds[k], bounds[k + 1]); it is
// uploaded on s_in into one of two input buffers of in_bytes, run on the context's stream into one of `ring` output
// slots of out_bytes (at most one per chunk) and downloaded on s_out as one copy: bytes [out_at(c0), out_at(c1)) of y.
// zero(c0, c1): the chunk's slot is zeroed before its run (whole padded rows, of which a row past its utterance's y_len
// reads as zero on the host).  upload(p, u0, m, in) enqueues the copies of the chunk of utterances u0 .. u0 + m with
// p.h2d; run(u0, m, in, out) enqueues its work.  Both runners synchronise the host with the device inside a run (pulse
// counts), so the upload of chunk k + 1 is enqueued before chunk k runs: it then overlaps chunk k's kernels instead of
// following the host's wait.
template <class Upload, class Run, class OutAt, class Zero>
int chunk_pipeline(WorldB200 *h, const char *who, const std::vector<int> &bounds, int ring, size_t in_bytes,
                   size_t out_bytes, OutAt out_at, Zero zero, int nbit, void *y, Upload upload, Run run) {
  Ctx *ctx = &h->c;
  const int n_chunks = (int)bounds.size() - 1, n_utts = bounds.back();
  int chunk = 0;
  for (int k = 0; k < n_chunks; ++k) chunk = imax(chunk, bounds[k + 1] - bounds[k]);
  ring = imin(ring, n_chunks);
  enum { EV_IN = 0, EV_CDONE = 2, EV_OUT = 4 };   // two input buffers, then `ring` output slots
  HostPipe p(h, who);
  int rc = p.open(EV_OUT + ring);
  if (rc) return rc;
  unsigned char *din[2] = {nullptr, nullptr};
  std::vector<unsigned char *> dout(ring, nullptr);
  for (int i = 0; i < (n_chunks > 1 ? 2 : 1) && !rc; ++i) rc = p.buffer(in_bytes, &din[i]);
  for (int i = 0; i < ring && !rc; ++i) rc = p.buffer(out_bytes, &dout[i]);
  auto upload_chunk = [&](int k) {
    if (k >= 2) p.wait(HostPipe::IN, EV_CDONE + (k & 1));   // the kernels of chunk k-2 have read din[k & 1]
    upload(p, bounds[k], bounds[k + 1] - bounds[k], din[k & 1]);
    p.record(EV_IN + (k & 1), HostPipe::IN);
    p.mark("h2d_done", k, HostPipe::IN);
  };
  if (!rc) upload_chunk(0);
  for (int k = 0; k < n_chunks && !rc; ++k) {
    const int u0 = bounds[k], m = bounds[k + 1] - u0, s = k & 1, slot = k % ring;
    const size_t o0 = out_at(u0), o1 = out_at(u0 + m);
    if (k + 1 < n_chunks) upload_chunk(k + 1);
    p.wait(HostPipe::RUN, EV_IN + s);
    if (k >= ring) p.wait(HostPipe::RUN, EV_OUT + slot);   // the slot's previous chunk is on the host
    p.mark("run_begin", k, HostPipe::RUN);
    if (zero(u0, u0 + m)) rc = dev_memset(ctx, dout[slot], 0, o1 - o0);
    if (!rc) rc = run(u0, m, din[s], dout[slot]);
    if (rc) break;
    p.record(EV_CDONE + s, HostPipe::RUN);   // behind chunk k's last kernel
    p.mark("run_end", k, HostPipe::RUN);
    p.wait(HostPipe::OUT, EV_CDONE + s);
    p.d2h((unsigned char *)y + o0, dout[slot], o1 - o0);
    p.record(EV_OUT + slot, HostPipe::OUT);
    p.mark("d2h_end", k, HostPipe::OUT);
  }
  char header[128];
  snprintf(header, sizeof header, "%s chunk %d chunks %d ring %d n %d nbit %d", who, chunk, n_chunks, ring, n_utts,
           nbit);
  rc = p.finish(rc, header);
  if (!rc) rc = world_b200_synchronize(h);
  return rc;
}

// chunk_pipeline's chunks of `chunk` utterances (the last one shorter), their outputs whole rows of `row` bytes, and
// whether a chunk's rows need zeroing: a row past its utterance's y_len
std::vector<int> even_bounds(int n_utts, int chunk) {
  std::vector<int> b;
  for (int u = 0; u < n_utts; u += chunk) b.push_back(u);
  b.push_back(n_utts);
  return b;
}
auto padded_at(size_t row) {
  return [row](int u) { return (size_t)u * row; };
}
auto ragged_rows(const int *y_len, int y_stride) {
  return [y_len, y_stride](int c0, int c1) {
    for (int u = c0; u < c1; ++u)
      if (y_len[u] != y_stride) return true;
    return false;
  };
}

// Synthesis from coded rows for host arrays: f0 + coded rows in, synthesis_run on each chunk, waveforms out, through
// chunk_pipeline with an output ring of three chunks.  A chunk is one pass of synthesis_run: a longer chunk would
// hold its download until all its passes were done, and a shorter one would pay the pass's fixed cost more often
// (syn_timebase_kernel's sequential phase sum over each utterance takes about as long for a few utterances as for a
// pass of hundreds; at 1024 x 10 s, 16 kHz, chunks of 128 utterances made the call slower than the serial path).  Two
// input sets and the output ring stay within a third of the scratch budget.  `host`: the call's host rows.
int synthesis_pipeline(WorldB200 *h, const SynthesisPlan &plan, const SynthesisRows &host) {
  Ctx *ctx = &h->c;
  const int n_utts = plan.n, f0_stride = plan.f0_stride, dims = plan.dims, n_ap = plan.n_ap;
  const size_t out_bytes = plan.nbit ? 2 : 8;
  const size_t per_in = (size_t)f0_stride * (1 + dims + n_ap) * 8, per_out = (size_t)plan.y_stride * out_bytes;
  int max_y = 0;
  for (const int v : plan.y_len) max_y = imax(max_y, v);
  const SynthesisSizing sz(ctx, plan, max_y);
  const int ring = 3;
  const size_t third = ctx->scratch_budget / 3;
  int chunk = imax(1, sz.fit(sz.nominal_cap));
  chunk = imin(chunk, (int)dmax(1.0, (double)third / (double)(2 * per_in + ring * per_out)));
  chunk = balanced_chunk(n_utts, chunk);
  ArenaPlan in_plan;
  const size_t o_f0 = in_plan.add((size_t)chunk * f0_stride * 8);
  const size_t o_sp = in_plan.add((size_t)chunk * f0_stride * dims * 8);
  const size_t o_ap = in_plan.add((size_t)chunk * f0_stride * n_ap * 8);
  // chunk k's f0 and coded rows
  auto upload = [&](HostPipe &p, int u0, int m, unsigned char *d) {
    const size_t frames = (size_t)m * f0_stride, row0 = (size_t)u0 * f0_stride;
    p.h2d(d + o_f0, host.f0 + row0, frames * 8);
    p.h2d(d + o_sp, host.sp + row0 * dims, frames * dims * 8);
    if (n_ap) p.h2d(d + o_ap, host.ap + row0 * n_ap, frames * n_ap * 8);
  };
  auto run = [&](int u0, int m, unsigned char *d, unsigned char *out) {
    return synthesis_run(ctx, plan, u0, m, {(const double *)(d + o_f0), (const double *)(d + o_sp),
                                            (const double *)(d + o_ap), out});
  };
  return chunk_pipeline(h, "synthesis", even_bounds(n_utts, chunk), ring, in_plan.total, (size_t)chunk * per_out,
                        padded_at(per_out), ragged_rows(plan.y_len.data(), plan.y_stride), plan.nbit, host.y, upload,
                        run);
}

// The packed form for host arrays: chunk k is utterances [c0, c1) whose frames [f_off[c0], f_off[c1]) of each input array
// go up as one copy and whose samples [y_off[c0], y_off[c1]) come back as one copy.  A chunk is one packed pass of
// synthesis_run (at most WB_HOST_CHUNK utterances when that is set), and two input sets and the output ring stay within
// a third of the scratch budget.
int synthesis_packed_pipeline(WorldB200 *h, const SynthesisPlan &plan, const SynthesisRows &host) {
  Ctx *ctx = &h->c;
  const int n_utts = plan.n, dims = plan.dims, n_ap = plan.n_ap;
  const long long *fo = plan.f_off.data(), *yo = plan.y_off.data();
  const size_t out_bytes = plan.nbit ? 2 : 8, per_frame = (size_t)(1 + dims + n_ap) * 8;
  const SynthesisSizing sz(ctx, plan, plan.y_stride);
  const int ring = 3;
  const double third = (double)(ctx->scratch_budget / 3);
  int most = 65535;
  if (const char *e = getenv("WB_HOST_CHUNK")) most = atoi(e) > 0 ? imin(most, atoi(e)) : most;
  std::vector<int> bounds{0};
  size_t most_frames = 0, most_samples = 0;
  while (bounds.back() < n_utts) {
    const int c0 = bounds.back();
    double pass = (double)sz.packed_pass();
    int c1 = c0;
    while (c1 < n_utts && c1 - c0 < most) {
      const double next = pass + (double)sz.packed_utt(plan.y_len[c1], plan.f_len[c1], sz.cap_of(plan.y_len[c1]));
      const double io = 2.0 * (double)(fo[c1 + 1] - fo[c0]) * per_frame + ring * (double)(yo[c1 + 1] - yo[c0]) * out_bytes;
      if (c1 > c0 && (next > sz.budget || io > third)) break;
      pass = next;
      ++c1;
    }
    bounds.push_back(c1);
    most_frames = std::max(most_frames, (size_t)(fo[c1] - fo[c0]));
    most_samples = std::max(most_samples, (size_t)(yo[c1] - yo[c0]));
  }
  ArenaPlan in_plan;
  const size_t o_f0 = in_plan.add(most_frames * 8);
  const size_t o_sp = in_plan.add(most_frames * dims * 8);
  const size_t o_ap = in_plan.add(most_frames * n_ap * 8);
  // the chunk's frames of f0 and of the coded rows, one copy each
  auto upload = [&](HostPipe &p, int u0, int m, unsigned char *d) {
    const size_t frames = (size_t)(fo[u0 + m] - fo[u0]), f0 = (size_t)fo[u0];
    p.h2d(d + o_f0, host.f0 + f0, frames * 8);
    p.h2d(d + o_sp, host.sp + f0 * dims, frames * dims * 8);
    if (n_ap) p.h2d(d + o_ap, host.ap + f0 * n_ap, frames * n_ap * 8);
  };
  auto run = [&](int u0, int m, unsigned char *d, unsigned char *out) {
    return synthesis_run(ctx, plan, u0, m, {(const double *)(d + o_f0), (const double *)(d + o_sp),
                                            (const double *)(d + o_ap), out});
  };
  auto out_at = [&](int u) { return (size_t)yo[u] * out_bytes; };
  auto zero = [](int, int) { return false; };   // every sample of the chunk is written
  return chunk_pipeline(h, "synthesis_packed", bounds, ring, in_plan.total, most_samples * out_bytes, out_at, zero,
                        plan.nbit, host.y, upload, run);
}

// Voice transformation for host arrays: chunks of PCM in, transform_run on each chunk (which forks from and joins back
// to the context's stream), output rows out, through chunk_pipeline with two output slots.  Chunks of WB_HOST_CHUNK
// utterances (default 512), fewer when the four buffers would take more than a sixth of the scratch budget.
int transform_pipeline(WorldB200 *h, const ChainRequest &r, const TransformPlan &tp, void *y) {
  Ctx *ctx = &h->c;
  const int n_utts = r.n;
  const size_t per_in = (size_t)r.x_stride * (r.nbit ? r.nbit / 8 : 8);
  const size_t per_out = (size_t)tp.syn.y_stride * (tp.syn.nbit ? 2 : 8);
  int chunk = 512;
  if (const char *e = getenv("WB_HOST_CHUNK")) chunk = atoi(e) > 0 ? atoi(e) : chunk;
  chunk = imin(chunk, (int)dmax(1.0, (double)(ctx->scratch_budget / 6) / (double)(2 * (per_in + per_out))));
  chunk = balanced_chunk(n_utts, chunk);
  // chunk k's PCM rows
  auto upload = [&](HostPipe &p, int u0, int m, unsigned char *d) {
    p.h2d(d, (const unsigned char *)r.x + (size_t)u0 * per_in, (size_t)m * per_in);
  };
  auto run = [&](int u0, int m, unsigned char *d, unsigned char *out) {
    return transform_run(h, r, tp, d, u0, m, out);
  };
  return chunk_pipeline(h, "transform", even_bounds(n_utts, chunk), 2, (size_t)chunk * per_in, (size_t)chunk * per_out,
                        padded_at(per_out), ragged_rows(tp.syn.y_len.data(), tp.syn.y_stride), tp.syn.nbit, y, upload,
                        run);
}

// The packed form for host arrays: chunks of consecutive utterances (at most WB_HOST_CHUNK, default 512, fewer when two
// input and two output buffers would take more than a sixth of the scratch budget).  Chunk k's samples
// [x_offsets[c0], x_offsets[c1]) go up as one copy, transform_run transforms them, and its samples [y_off[c0],
// y_off[c1]) come back as one copy; every sample of a chunk is written, so nothing is zeroed.
// cv: HOST curves on the analysis frames (world_b200_transform_host_packed_curves); each chunk's curve frames
// [f_off[c0], f_off[c1]) go up as one copy per curve after its samples, in the same input buffer.
int transform_packed_pipeline(WorldB200 *h, const ChainRequest &r, const TransformPlan &tp, void *y,
                              const ModifyCurves *cv = nullptr) {
  Ctx *ctx = &h->c;
  const int n_utts = r.n;
  const long long *xo = r.x_offsets, *yo = tp.syn.y_off.data(), *fo = tp.chain.f_off.data();
  const size_t in_bytes = r.nbit ? (size_t)(r.nbit / 8) : 8, out_bytes = tp.syn.nbit ? 2 : 8;
  const size_t curve_bytes = cv ? 8 * ((cv->f0 ? 1 : 0) + (cv->ratio ? 1 : 0)) : 0;   // per frame
  int most = 512;
  if (const char *e = getenv("WB_HOST_CHUNK")) most = atoi(e) > 0 ? atoi(e) : most;
  const size_t cap = ctx->scratch_budget / 6;
  auto bytes = [&](int c0, int c1) {
    return 2 * ((size_t)(xo[c1] - xo[c0]) * in_bytes + (size_t)(yo[c1] - yo[c0]) * out_bytes +
                (size_t)(fo[c1] - fo[c0]) * curve_bytes);
  };
  std::vector<int> bounds{0};
  size_t most_in = 0, most_out = 0, most_frames = 0;
  while (bounds.back() < n_utts) {
    const int c0 = bounds.back();
    int c1 = c0 + 1;
    while (c1 < n_utts && c1 - c0 < most && bytes(c0, c1 + 1) <= cap) ++c1;
    bounds.push_back(c1);
    most_in = std::max(most_in, (size_t)(xo[c1] - xo[c0]) * in_bytes);
    most_out = std::max(most_out, (size_t)(yo[c1] - yo[c0]) * out_bytes);
    most_frames = std::max(most_frames, (size_t)(fo[c1] - fo[c0]));
  }
  ArenaPlan in_plan;
  in_plan.add(most_in);
  const size_t o_f0 = in_plan.add(cv && cv->f0 ? most_frames * 8 : 0);
  const size_t o_ratio = in_plan.add(cv && cv->ratio ? most_frames * 8 : 0);
  // chunk k's samples, one copy, and its frames of each curve, one copy each
  auto upload = [&](HostPipe &p, int u0, int m, unsigned char *d) {
    p.h2d(d, (const unsigned char *)r.x + (size_t)xo[u0] * in_bytes, (size_t)(xo[u0 + m] - xo[u0]) * in_bytes);
    const size_t frames = (size_t)(fo[u0 + m] - fo[u0]);
    if (cv && cv->f0) p.h2d(d + o_f0, cv->f0 + fo[u0], frames * 8);
    if (cv && cv->ratio) p.h2d(d + o_ratio, cv->ratio + fo[u0], frames * 8);
  };
  auto run = [&](int u0, int m, unsigned char *d, unsigned char *out) {
    if (!cv) return transform_run(h, r, tp, d, u0, m, out);
    ModifyCurves dc;
    dc.f0 = cv->f0 ? (const double *)(d + o_f0) : nullptr;
    dc.ratio = cv->ratio ? (const double *)(d + o_ratio) : nullptr;
    return transform_run(h, r, tp, d, u0, m, out, &dc);
  };
  auto out_at = [&](int u) { return (size_t)yo[u] * out_bytes; };
  auto zero = [](int, int) { return false; };
  return chunk_pipeline(h, "transform_packed", bounds, 2, in_plan.total, most_out, out_at, zero, tp.syn.nbit, y, upload,
                        run);
}

// world_b200_synthesis_coded_host and, with f0_scale / spectral_ratio, world_b200_synthesis_coded_host_modified: every
// check runs before the first chunk is queued
// (fft_sizes NULL: fft_size for every utterance; world_b200_synthesis_coded_host_options passes per_utt)
int synthesis_coded_host(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts, int f0_stride,
                         const double *coded_spectral_envelope, int number_of_dimensions,
                         const double *coded_aperiodicity, int fft_size, double frame_period, int fs,
                         const int *y_lengths, int y_stride, int nbit, void *y, const double *f0_scale,
                         const double *spectral_ratio, bool per_utt = false, const int *fft_sizes = nullptr) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  SynthesisRequest r{f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, coded_aperiodicity, fft_size,
                     frame_period, fs, y_lengths, y_stride, y, nbit};
  r.coded = true; r.dims = number_of_dimensions; r.f0_scale = f0_scale; r.spectral_ratio = spectral_ratio;
  r.per_utt = per_utt; r.fft_sizes = fft_sizes;
  SynthesisPlan plan;
  const int rc = synthesis_plan(&h->c, r, "Synthesis", &plan);
  if (rc || n_utts == 0) return rc;
  return synthesis_pipeline(h, plan, {r.f0, r.sp, r.ap, r.y});
}

}  // namespace

extern "C" int world_b200_synthesis_coded_host_packed(WorldB200 *h, const double *f0, int n_utts,
                                                      const long long *f_offsets,
                                                      const double *coded_spectral_envelope, int number_of_dimensions,
                                                      const double *coded_aperiodicity, const int *fft_sizes,
                                                      double frame_period, int fs, const long long *y_offsets,
                                                      const double *f0_scale, const double *spectral_ratio, int nbit,
                                                      void *y) {
  if (!h) return WORLD_B200_EINVAL;
  if (n_utts == 0) return 0;
  DeviceGuard guard_(&h->c);
  if (!f_offsets || !y_offsets) {
    h->c.last_error = "Synthesis: f_offsets and y_offsets must be given";
    return WORLD_B200_EINVAL;
  }
  SynthesisRequest r{f0, nullptr, n_utts, 0, coded_spectral_envelope, coded_aperiodicity, 0, frame_period, fs, nullptr,
                     0, y, nbit};
  r.coded = true; r.dims = number_of_dimensions; r.f0_scale = f0_scale; r.spectral_ratio = spectral_ratio;
  r.per_utt = true; r.fft_sizes = fft_sizes; r.f_offsets = f_offsets; r.y_offsets = y_offsets;
  SynthesisPlan plan;
  const int rc = synthesis_plan(&h->c, r, "Synthesis", &plan);
  return rc ? rc : synthesis_packed_pipeline(h, plan, {r.f0, r.sp, r.ap, r.y});
}

extern "C" int world_b200_synthesis_coded_host(WorldB200 *h, const double *f0, const int *f0_lengths, int n_utts,
                                               int f0_stride, const double *coded_spectral_envelope,
                                               int number_of_dimensions, const double *coded_aperiodicity,
                                               int fft_size, double frame_period, int fs, const int *y_lengths,
                                               int y_stride, int nbit, void *y) {
  return synthesis_coded_host(h, f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, number_of_dimensions,
                              coded_aperiodicity, fft_size, frame_period, fs, y_lengths, y_stride, nbit, y, nullptr,
                              nullptr);
}

extern "C" int world_b200_synthesis_coded_host_modified(WorldB200 *h, const double *f0, const int *f0_lengths,
                                                        int n_utts, int f0_stride,
                                                        const double *coded_spectral_envelope,
                                                        int number_of_dimensions, const double *coded_aperiodicity,
                                                        int fft_size, double frame_period, int fs,
                                                        const int *y_lengths, int y_stride, const double *f0_scale,
                                                        const double *spectral_ratio, int nbit, void *y) {
  return synthesis_coded_host(h, f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, number_of_dimensions,
                              coded_aperiodicity, fft_size, frame_period, fs, y_lengths, y_stride, nbit, y, f0_scale,
                              spectral_ratio);
}

extern "C" int world_b200_synthesis_coded_host_options(WorldB200 *h, const double *f0, const int *f0_lengths,
                                                       int n_utts, int f0_stride,
                                                       const double *coded_spectral_envelope,
                                                       int number_of_dimensions, const double *coded_aperiodicity,
                                                       const int *fft_sizes, double frame_period, int fs,
                                                       const int *y_lengths, int y_stride, const double *f0_scale,
                                                       const double *spectral_ratio, int nbit, void *y) {
  return synthesis_coded_host(h, f0, f0_lengths, n_utts, f0_stride, coded_spectral_envelope, number_of_dimensions,
                              coded_aperiodicity, 0, frame_period, fs, y_lengths, y_stride, nbit, y, f0_scale,
                              spectral_ratio, true, fft_sizes);
}

extern "C" int world_b200_transform_host_spectral_options(
    WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths, int fs,
    const WorldB200AnalysisOption *option, const HarvestOption *harvest_options, const DioOption *dio_options,
    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options, const double *f0_scale,
    const double *spectral_ratio, const double *time_scale, int nbit_out, void *y, int y_stride, int *y_lengths) {
  if (!h) return WORLD_B200_EINVAL;
  DeviceGuard guard_(&h->c);
  ChainRequest r(x, nbit, n_utts, x_stride, x_lengths, fs, option, nullptr, nullptr, 0, nullptr, nullptr);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options;
  r.transform = true;
  TransformPlan tp;
  const int rc = transform_check(h, r, f0_scale, spectral_ratio, time_scale, nbit_out, y, y_stride, "transform_host", &tp);
  if (rc) return rc;
  if (y_lengths) std::copy(tp.syn.y_len.begin(), tp.syn.y_len.end(), y_lengths);
  if (n_utts == 0) return 0;
  return transform_pipeline(h, r, tp, y);
}

extern "C" int world_b200_transform_host(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride,
                                         const int *x_lengths, int fs, const WorldB200AnalysisOption *option,
                                         const HarvestOption *harvest_options, const DioOption *dio_options,
                                         const double *f0_scale, const double *spectral_ratio,
                                         const double *time_scale, int nbit_out, void *y, int y_stride,
                                         int *y_lengths) {
  return world_b200_transform_host_spectral_options(h, x, nbit, n_utts, x_stride, x_lengths, fs, option,
                                                    harvest_options, dio_options, nullptr, nullptr, f0_scale,
                                                    spectral_ratio, time_scale, nbit_out, y, y_stride, y_lengths);
}

extern "C" int world_b200_transform_host_packed(WorldB200 *h, const void *x, int nbit, int n_utts,
                                                const long long *x_offsets, int fs,
                                                const WorldB200AnalysisOption *option,
                                                const HarvestOption *harvest_options, const DioOption *dio_options,
                                                const CheapTrickOption *cheaptrick_options,
                                                const D4COption *d4c_options, const double *f0_scale,
                                                const double *spectral_ratio, const double *time_scale, int nbit_out,
                                                void *y, long long *y_offsets) {
  if (!h) return WORLD_B200_EINVAL;
  if (n_utts == 0) {
    if (y_offsets) y_offsets[0] = 0;
    return 0;
  }
  DeviceGuard guard_(&h->c);
  ChainRequest r = packed_request(x, nbit, n_utts, x_offsets, fs, option, harvest_options, dio_options,
                                  cheaptrick_options, d4c_options, nullptr, nullptr, nullptr, nullptr);
  r.transform = true;
  TransformPlan tp;
  const int rc = transform_check(h, r, f0_scale, spectral_ratio, time_scale, nbit_out, y, 0, "transform_host_packed",
                                 &tp);
  if (rc) return rc;
  if (y_offsets) std::copy(tp.syn.y_off.begin(), tp.syn.y_off.end(), y_offsets);
  return transform_packed_pipeline(h, r, tp, y);
}

extern "C" int world_b200_transform_host_packed_curves(WorldB200 *h, const void *x, int nbit, int n_utts,
                                                       const long long *x_offsets, int fs,
                                                       const WorldB200AnalysisOption *option,
                                                       const HarvestOption *harvest_options,
                                                       const DioOption *dio_options,
                                                       const CheapTrickOption *cheaptrick_options,
                                                       const D4COption *d4c_options, const double *f0_curve,
                                                       const double *spectral_ratio_curve, const double *time_scale,
                                                       int nbit_out, void *y, long long *y_offsets) {
  if (!h) return WORLD_B200_EINVAL;
  if (n_utts == 0) {
    if (y_offsets) y_offsets[0] = 0;
    return 0;
  }
  DeviceGuard guard_(&h->c);
  ChainRequest r = packed_request(x, nbit, n_utts, x_offsets, fs, option, harvest_options, dio_options,
                                  cheaptrick_options, d4c_options, nullptr, nullptr, nullptr, nullptr);
  r.transform = true;
  TransformPlan tp;
  const char *who = "transform_host_packed_curves";
  ModifyCurves cv;
  cv.f0 = f0_curve; cv.ratio = spectral_ratio_curve;
  int rc = transform_check(h, r, nullptr, nullptr, time_scale, nbit_out, y, 0, who, &tp);
  const ChainPlan &p = tp.chain;
  if (!rc) rc = curves_check_host(&h->c, who, cv, n_utts, p.f_len.data(), 0, p.f_off.data(), p.ct.fft_size.data());
  if (rc) return rc;
  if (y_offsets) std::copy(tp.syn.y_off.begin(), tp.syn.y_off.end(), y_offsets);
  return transform_packed_pipeline(h, r, tp, y, &cv);
}

extern "C" int world_b200_analyze_host(WorldB200 *h, const double *x, int n_utts, int x_stride,
                                       const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                       double *time_axis, double *f0, int f0_stride, double *spectrogram,
                                       double *aperiodicity) {
  return analyze_pipeline(h, ChainRequest(x, 0, n_utts, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride,
                                          spectrogram, aperiodicity));
}

extern "C" int world_b200_analyze_host_options(WorldB200 *h, const double *x, int n_utts, int x_stride,
                                               const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                               const HarvestOption *harvest_options, double *time_axis, double *f0,
                                               int f0_stride, double *spectrogram, double *aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  ChainRequest r(x, 0, n_utts, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram, aperiodicity);
  r.harvest_options = harvest_options;
  return analyze_pipeline(h, r);
}

extern "C" int world_b200_analyze_host_dio_options(WorldB200 *h, const double *x, int n_utts, int x_stride,
                                                   const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                   const DioOption *dio_options, double *time_axis, double *f0,
                                                   int f0_stride, double *spectrogram, double *aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  ChainRequest r(x, 0, n_utts, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram, aperiodicity);
  r.dio_options = dio_options;
  return analyze_pipeline(h, r);
}

// analyze_host with per-utterance CheapTrick / D4C options (either array may be NULL), F0 options as above, and full
// rows of row_stride doubles per frame
extern "C" int world_b200_analyze_host_spectral_options(
    WorldB200 *h, const double *x, int n_utts, int x_stride, const int *x_lengths, int fs,
    const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options, const DioOption *dio_options,
    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options, double *time_axis, double *f0,
    int f0_stride, int row_stride, double *spectrogram, double *aperiodicity) {
  ChainRequest r(x, 0, n_utts, x_stride, x_lengths, fs, opt, time_axis, f0, f0_stride, spectrogram, aperiodicity);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options; r.row_stride = row_stride;
  return analyze_pipeline(h, r);
}

extern "C" int world_b200_analyze_host_packed(WorldB200 *h, const double *x, int n_utts, const long long *x_offsets,
                                              int fs, const WorldB200AnalysisOption *opt,
                                              const HarvestOption *harvest_options, const DioOption *dio_options,
                                              const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options,
                                              double *time_axis, double *f0, int row_stride, double *spectrogram,
                                              double *aperiodicity, long long *f_offsets) {
  ChainRequest r = packed_request(x, 0, n_utts, x_offsets, fs, opt, harvest_options, dio_options, cheaptrick_options,
                                  d4c_options, time_axis, f0, spectrogram, aperiodicity);
  r.row_stride = row_stride;
  return analyze_packed_pipeline(h, r, f_offsets);
}

extern "C" int world_b200_analyze_coded_host_packed(
    WorldB200 *h, const void *x, int nbit, int n_utts, const long long *x_offsets, int fs,
    const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options, const DioOption *dio_options,
    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options, int number_of_dimensions,
    double *time_axis, double *f0, double *coded_spectral_envelope, double *coded_aperiodicity, long long *f_offsets) {
  ChainRequest r = packed_request(x, nbit, n_utts, x_offsets, fs, opt, harvest_options, dio_options, cheaptrick_options,
                                  d4c_options, time_axis, f0, coded_spectral_envelope, coded_aperiodicity);
  r.coded = true; r.dims = number_of_dimensions;
  return analyze_packed_pipeline(h, r, f_offsets);
}

// analyze_coded_host with per-utterance CheapTrick / D4C options (either array may be NULL) and F0 options as above
extern "C" int world_b200_analyze_coded_host_spectral_options(
    WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride, const int *x_lengths, int fs,
    const WorldB200AnalysisOption *opt, const HarvestOption *harvest_options, const DioOption *dio_options,
    const CheapTrickOption *cheaptrick_options, const D4COption *d4c_options, int number_of_dimensions,
    double *time_axis, double *f0, int f0_stride, double *coded_spectral_envelope, double *coded_aperiodicity) {
  ChainRequest r = coded_request(x, nbit, n_utts, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                 f0_stride, coded_spectral_envelope, coded_aperiodicity);
  r.harvest_options = harvest_options; r.dio_options = dio_options;
  r.cheaptrick_options = cheaptrick_options; r.d4c_options = d4c_options;
  return analyze_pipeline(h, r);
}

extern "C" int world_b200_analyze_coded_host(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride,
                                             const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                             int number_of_dimensions, double *time_axis, double *f0, int f0_stride,
                                             double *coded_spectral_envelope, double *coded_aperiodicity) {
  return analyze_pipeline(h, coded_request(x, nbit, n_utts, x_stride, x_lengths, fs, opt, number_of_dimensions,
                                           time_axis, f0, f0_stride, coded_spectral_envelope, coded_aperiodicity));
}

extern "C" int world_b200_analyze_coded_host_options(WorldB200 *h, const void *x, int nbit, int n_utts, int x_stride,
                                                     const int *x_lengths, int fs, const WorldB200AnalysisOption *opt,
                                                     const HarvestOption *harvest_options, int number_of_dimensions,
                                                     double *time_axis, double *f0, int f0_stride,
                                                     double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!harvest_options) return WORLD_B200_EINVAL;
  ChainRequest r = coded_request(x, nbit, n_utts, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                 f0_stride, coded_spectral_envelope, coded_aperiodicity);
  r.harvest_options = harvest_options;
  return analyze_pipeline(h, r);
}

extern "C" int world_b200_analyze_coded_host_dio_options(WorldB200 *h, const void *x, int nbit, int n_utts,
                                                         int x_stride, const int *x_lengths, int fs,
                                                         const WorldB200AnalysisOption *opt,
                                                         const DioOption *dio_options, int number_of_dimensions,
                                                         double *time_axis, double *f0, int f0_stride,
                                                         double *coded_spectral_envelope, double *coded_aperiodicity) {
  if (!dio_options) return WORLD_B200_EINVAL;
  ChainRequest r = coded_request(x, nbit, n_utts, x_stride, x_lengths, fs, opt, number_of_dimensions, time_axis, f0,
                                 f0_stride, coded_spectral_envelope, coded_aperiodicity);
  r.dio_options = dio_options;
  return analyze_pipeline(h, r);
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
    ctx = h ? &h->c : nullptr;
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
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
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
  DeviceGuard guard_(&h->c);
  Ctx *ctx = &h->c;
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
