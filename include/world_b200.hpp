// world_b200.hpp -- C++ batched overloads of the reference's entry points.
//
// BASELINE.json's north_star: "Dio()/Harvest()/StoneMask()/CheapTrick()/D4C()/Synthesis() ... stay
// source-compatible and gain batched overloads that take N waveforms at once".  The C symbols of
// include/world/*.h cannot be overloaded, so the overloads live here, outside any extern "C" block
// (SURVEY.md 8b), header-only on top of the C ABI of world_b200.h.  They keep the reference's calling
// convention -- the caller owns every buffer, one pointer per utterance, `double **` rows for the
// spectrogram / aperiodicity -- and add a leading `n_utts`:
//
//   Dio(xs, x_lengths, n_utts, fs, &option, temporal_positions, f0s);
//   CheapTrick(xs, x_lengths, n_utts, fs, temporal_positions, f0s, f0_lengths, &option, spectrograms);
//
// Each call packs the utterances into one padded batch, runs the batched kernels on the GPU of a
// process-wide context (device $WORLD_B200_DEVICE, default 0) and scatters the results back.
// They return the library's status code (0 = success) instead of void.
#ifndef WORLD_B200_HPP_
#define WORLD_B200_HPP_

#include <cuda_runtime_api.h>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "world_b200.h"

namespace world_b200 {

inline WorldB200 *shared_context() {
  static WorldB200 *ctx = nullptr;
  if (!ctx) {
    int dev = 0;
    if (const char *e = std::getenv("WORLD_B200_DEVICE")) dev = std::atoi(e);
    if (world_b200_create(dev, &ctx) != 0) ctx = nullptr;
  }
  return ctx;
}

// RAII device buffer (plain cudaMalloc; these helpers are conveniences, not the fast path)
struct DeviceArray {
  double *p = nullptr;
  explicit DeviceArray(size_t n) { if (cudaMalloc(reinterpret_cast<void **>(&p), (n ? n : 1) * sizeof(double)) != cudaSuccess) p = nullptr; }
  ~DeviceArray() { if (p) cudaFree(p); }
  DeviceArray(const DeviceArray &) = delete;
  DeviceArray &operator=(const DeviceArray &) = delete;
};

inline int max_of(const int *v, int n) { int m = 0; for (int i = 0; i < n; ++i) if (v[i] > m) m = v[i]; return m; }

// pack n host vectors of different lengths into one padded host matrix
inline std::vector<double> pack(const double *const *rows, const int *lengths, int n, int stride) {
  std::vector<double> m(static_cast<size_t>(n) * stride, 0.0);
  for (int i = 0; i < n; ++i) std::memcpy(m.data() + static_cast<size_t>(i) * stride, rows[i], sizeof(double) * lengths[i]);
  return m;
}

inline int upload(DeviceArray &d, const std::vector<double> &h) {
  return d.p && cudaMemcpy(d.p, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice) == cudaSuccess ? 0 : WORLD_B200_ECUDA;
}

inline int download_rows(const DeviceArray &d, int n, int stride, const int *lengths, double *const *rows) {
  std::vector<double> h(static_cast<size_t>(n) * stride);
  if (cudaMemcpy(h.data(), d.p, h.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) return WORLD_B200_ECUDA;
  for (int i = 0; i < n; ++i) std::memcpy(rows[i], h.data() + static_cast<size_t>(i) * stride, sizeof(double) * lengths[i]);
  return 0;
}

inline int download_frames(const DeviceArray &d, int n, int f_stride, int bins, const int *f0_lengths, double **const *out) {
  std::vector<double> h(static_cast<size_t>(n) * f_stride * bins);
  if (cudaMemcpy(h.data(), d.p, h.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) return WORLD_B200_ECUDA;
  for (int u = 0; u < n; ++u)
    for (int i = 0; i < f0_lengths[u]; ++i)
      std::memcpy(out[u][i], h.data() + (static_cast<size_t>(u) * f_stride + i) * bins, sizeof(double) * bins);
  return 0;
}

inline std::vector<int> frame_counts(const int *x_lengths, int n, int fs, double frame_period) {
  std::vector<int> fl(n);
  for (int i = 0; i < n; ++i) fl[i] = world_b200_frames(fs, x_lengths[i], frame_period);
  return fl;
}

}  // namespace world_b200

// ---- batched overloads (same argument order as the single-utterance functions, plus n_utts) ----------

// Dio over N waveforms: temporal_positions[u] / f0s[u] hold GetSamplesForDIO(fs, x_lengths[u], ...) doubles.
inline int Dio(const double *const *xs, const int *x_lengths, int n_utts, int fs, const DioOption *option,
               double *const *temporal_positions, double *const *f0s) {
  using namespace world_b200;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts);
  const std::vector<int> fl = frame_counts(x_lengths, n_utts, fs, option->frame_period);
  const int f_stride = max_of(fl.data(), n_utts);
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = world_b200_dio_batch(w, dx.p, n_utts, xs_stride, x_lengths, fs, option, dt.p, df.p, f_stride);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_rows(dt, n_utts, f_stride, fl.data(), temporal_positions);
  if (!rc) rc = download_rows(df, n_utts, f_stride, fl.data(), f0s);
  return rc;
}

inline int Harvest(const double *const *xs, const int *x_lengths, int n_utts, int fs, const HarvestOption *option,
                   double *const *temporal_positions, double *const *f0s) {
  using namespace world_b200;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts);
  const std::vector<int> fl = frame_counts(x_lengths, n_utts, fs, option->frame_period);
  const int f_stride = max_of(fl.data(), n_utts);
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = world_b200_harvest_batch(w, dx.p, n_utts, xs_stride, x_lengths, fs, option, dt.p, df.p, f_stride);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_rows(dt, n_utts, f_stride, fl.data(), temporal_positions);
  if (!rc) rc = download_rows(df, n_utts, f_stride, fl.data(), f0s);
  return rc;
}

// One Harvest option per utterance (options.size() == n_utts): f0_floor / f0_ceil may differ, frame_period may not
// (world_b200_harvest_batch_options).  A vector, because a pointer would collide with the one-option overload above.
inline int Harvest(const double *const *xs, const int *x_lengths, int n_utts, int fs,
                   const std::vector<HarvestOption> &options, double *const *temporal_positions, double *const *f0s) {
  using namespace world_b200;
  if (n_utts < 0 || options.size() != static_cast<size_t>(n_utts)) return WORLD_B200_EINVAL;
  if (n_utts == 0) return 0;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts);
  const std::vector<int> fl = frame_counts(x_lengths, n_utts, fs, options[0].frame_period);
  const int f_stride = max_of(fl.data(), n_utts);
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = world_b200_harvest_batch_options(w, dx.p, n_utts, xs_stride, x_lengths, fs, options.data(), dt.p, df.p, f_stride);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_rows(dt, n_utts, f_stride, fl.data(), temporal_positions);
  if (!rc) rc = download_rows(df, n_utts, f_stride, fl.data(), f0s);
  return rc;
}

// One DIO option per utterance (options.size() == n_utts): f0_floor / f0_ceil / channels_in_octave / allowed_range may
// differ, frame_period and speed may not (world_b200_dio_batch_options).  A vector, as for Harvest above.
inline int Dio(const double *const *xs, const int *x_lengths, int n_utts, int fs, const std::vector<DioOption> &options,
               double *const *temporal_positions, double *const *f0s) {
  using namespace world_b200;
  if (n_utts < 0 || options.size() != static_cast<size_t>(n_utts)) return WORLD_B200_EINVAL;
  if (n_utts == 0) return 0;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts);
  const std::vector<int> fl = frame_counts(x_lengths, n_utts, fs, options[0].frame_period);
  const int f_stride = max_of(fl.data(), n_utts);
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = world_b200_dio_batch_options(w, dx.p, n_utts, xs_stride, x_lengths, fs, options.data(), dt.p, df.p, f_stride);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_rows(dt, n_utts, f_stride, fl.data(), temporal_positions);
  if (!rc) rc = download_rows(df, n_utts, f_stride, fl.data(), f0s);
  return rc;
}

inline int StoneMask(const double *const *xs, const int *x_lengths, int n_utts, int fs,
                     const double *const *temporal_positions, const double *const *f0s, const int *f0_lengths,
                     double *const *refined_f0s) {
  using namespace world_b200;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts), f_stride = max_of(f0_lengths, n_utts);
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = upload(dt, pack(temporal_positions, f0_lengths, n_utts, f_stride));
  if (!rc) rc = upload(df, pack(f0s, f0_lengths, n_utts, f_stride));
  if (!rc) rc = world_b200_stonemask_batch(w, dx.p, n_utts, xs_stride, x_lengths, fs, dt.p, df.p, f0_lengths, f_stride, df.p);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_rows(df, n_utts, f_stride, f0_lengths, refined_f0s);
  return rc;
}

// spectrograms[u][i] -> option->fft_size / 2 + 1 doubles (caller allocated), u < n_utts, i < f0_lengths[u]
inline int CheapTrick(const double *const *xs, const int *x_lengths, int n_utts, int fs,
                      const double *const *temporal_positions, const double *const *f0s, const int *f0_lengths,
                      const CheapTrickOption *option, double **const *spectrograms) {
  using namespace world_b200;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts), f_stride = max_of(f0_lengths, n_utts), bins = option->fft_size / 2 + 1;
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  DeviceArray ds(static_cast<size_t>(n_utts) * f_stride * bins);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = upload(dt, pack(temporal_positions, f0_lengths, n_utts, f_stride));
  if (!rc) rc = upload(df, pack(f0s, f0_lengths, n_utts, f_stride));
  if (!rc && !ds.p) rc = WORLD_B200_ENOMEM;
  if (!rc) rc = world_b200_cheaptrick_batch(w, dx.p, n_utts, xs_stride, x_lengths, fs, dt.p, df.p, f0_lengths, f_stride, option, ds.p);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_frames(ds, n_utts, f_stride, bins, f0_lengths, spectrograms);
  return rc;
}

inline int D4C(const double *const *xs, const int *x_lengths, int n_utts, int fs,
               const double *const *temporal_positions, const double *const *f0s, const int *f0_lengths, int fft_size,
               const D4COption *option, double **const *aperiodicities) {
  using namespace world_b200;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int xs_stride = max_of(x_lengths, n_utts), f_stride = max_of(f0_lengths, n_utts), bins = fft_size / 2 + 1;
  DeviceArray dx(static_cast<size_t>(n_utts) * xs_stride), dt(static_cast<size_t>(n_utts) * f_stride), df(static_cast<size_t>(n_utts) * f_stride);
  DeviceArray da(static_cast<size_t>(n_utts) * f_stride * bins);
  int rc = upload(dx, pack(xs, x_lengths, n_utts, xs_stride));
  if (!rc) rc = upload(dt, pack(temporal_positions, f0_lengths, n_utts, f_stride));
  if (!rc) rc = upload(df, pack(f0s, f0_lengths, n_utts, f_stride));
  if (!rc && !da.p) rc = WORLD_B200_ENOMEM;
  if (!rc) rc = world_b200_d4c_batch(w, dx.p, n_utts, xs_stride, x_lengths, fs, dt.p, df.p, f0_lengths, f_stride, fft_size, option, da.p);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_frames(da, n_utts, f_stride, bins, f0_lengths, aperiodicities);
  return rc;
}

// ys[u] -> y_lengths[u] doubles
inline int Synthesis(const double *const *f0s, const int *f0_lengths, int n_utts, const double *const *const *spectrograms,
                     const double *const *const *aperiodicities, int fft_size, double frame_period, int fs,
                     const int *y_lengths, double *const *ys) {
  using namespace world_b200;
  WorldB200 *w = shared_context();
  if (!w) return WORLD_B200_ECUDA;
  const int f_stride = max_of(f0_lengths, n_utts), y_stride = max_of(y_lengths, n_utts), bins = fft_size / 2 + 1;
  std::vector<double> hs(static_cast<size_t>(n_utts) * f_stride * bins, 1.0), ha(hs.size(), 1.0);
  for (int u = 0; u < n_utts; ++u)
    for (int i = 0; i < f0_lengths[u]; ++i) {
      std::memcpy(hs.data() + (static_cast<size_t>(u) * f_stride + i) * bins, spectrograms[u][i], sizeof(double) * bins);
      std::memcpy(ha.data() + (static_cast<size_t>(u) * f_stride + i) * bins, aperiodicities[u][i], sizeof(double) * bins);
    }
  DeviceArray df(static_cast<size_t>(n_utts) * f_stride), ds(hs.size()), da(ha.size()), dy(static_cast<size_t>(n_utts) * y_stride);
  int rc = upload(df, pack(f0s, f0_lengths, n_utts, f_stride));
  if (!rc) rc = upload(ds, hs);
  if (!rc) rc = upload(da, ha);
  if (!rc && !dy.p) rc = WORLD_B200_ENOMEM;
  if (!rc) rc = world_b200_synthesis_batch(w, df.p, f0_lengths, n_utts, f_stride, ds.p, da.p, fft_size, frame_period, fs, y_lengths, y_stride, dy.p);
  if (!rc) rc = world_b200_synchronize(w);
  if (!rc) rc = download_rows(dy, n_utts, y_stride, y_lengths, ys);
  return rc;
}

#endif  // WORLD_B200_HPP_
