// wb_block.cuh -- block-wide reductions / scans used by every frame kernel.
// All helpers need blockDim.x to be a multiple of 32 and must be called by every thread of
// the block (they contain barriers).  `red` is a shared scratch of >= 2*33 doubles.
// Results are deterministic (fixed combination order); they are NOT the reference's
// left-to-right order -- only sums that the survey measured as order-insensitive
// (SURVEY.md App. B4: everything except LinearSmoothing's running sum) go through here.
#pragma once
#include "wb_platform.cuh"

namespace wb {

#define WB_RED_DOUBLES 72

// The host emulation runs one thread per block; its reductions still store the partial sums where warp 0 of a CTA
// stores them (red[0], red[33], ...), so a kernel that keeps live data in `red` across a reduction fails there too.
WB_DEV double block_sum(double v, double *red) {
#ifdef WB_EMU
  red[0] = v;
  return red[0];
#else
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < nw; ++i) s += red[i];
  return s;
#endif
}

// two sums with one pair of barriers
WB_DEV void block_sum2(double &a, double &b, double *red) {
#ifdef WB_EMU
  red[0] = a; red[33] = b;
  a = red[0]; b = red[33];
#else
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) { red[w] = a; red[33 + w] = b; }
  __syncthreads();
  double sa = 0.0, sb = 0.0;
  for (int i = 0; i < nw; ++i) { sa += red[i]; sb += red[33 + i]; }
  a = sa; b = sb;
#endif
}

WB_DEV int block_sum_int(int v, double *red) {
#ifdef WB_EMU
  int *ired = reinterpret_cast<int *>(red);
  ired[0] = v;
  return ired[0];
#else
  int *ired = reinterpret_cast<int *>(red);
  v = __reduce_add_sync(0xffffffffu, v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) ired[w] = v;
  __syncthreads();
  int s = 0;
  for (int i = 0; i < nw; ++i) s += ired[i];
  return s;
#endif
}

// Inclusive prefix sum over a shared array a[0..n) in place (order: blocked tree, see header note).
// Each thread owns a contiguous chunk; chunk totals are scanned with warp shuffles.
// red_big: >= nthreads + 33 doubles of shared scratch.
WB_DEV void block_inclusive_scan(double *a, int n, double *red_big) {
  const int tid = WB_TID, nth = WB_NTH;
  const int chunk = (n + nth - 1) / nth;
  const int lo = imin(n, tid * chunk), hi = imin(n, lo + chunk);
  double s = 0.0;
  for (int i = lo; i < hi; ++i) { s += a[i]; a[i] = s; }
#ifdef WB_EMU
  (void)red_big;
#else
  // exclusive scan of the per-thread totals
  double inc = s;
  const int lane = tid & 31, w = tid >> 5, nw = (nth + 31) >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) red_big[w] = inc;
  __syncthreads();
  double base = inc - s;
  for (int i = 0; i < w && i < nw; ++i) base += red_big[i];
  if (base != 0.0 || tid > 0)
    for (int i = lo; i < hi; ++i) a[i] += base;
#endif
  WB_SYNC();
}

}  // namespace wb

namespace wb {
// K sums at once (K <= 8); red needs 33*K doubles -> use a scratch of WB_REDN_DOUBLES.
#define WB_REDN_DOUBLES (33 * 8)
template <int K>
WB_DEV void block_sum_n(double (&v)[K], double *red) {
#ifdef WB_EMU
  for (int k = 0; k < K; ++k) { red[33 * k] = v[k]; v[k] = red[33 * k]; }
#else
#pragma unroll
  for (int k = 0; k < K; ++k)
    for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) red[33 * k + w] = v[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double s = 0.0;
    for (int i = 0; i < nw; ++i) s += red[33 * k + i];
    v[k] = s;
  }
#endif
}
}  // namespace wb
