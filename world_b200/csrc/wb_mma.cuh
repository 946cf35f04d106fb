// wb_mma.cuh -- the FP64 tensor-core MMA (m16n8k8, DMMA) and the lane-generic idiom its host emulation needs.
#pragma once
#include "wb_platform.cuh"

// Lane-generic source: WB_FOR_LANES runs the lane body for lane = threadIdx.x & 31 on the GPU and for all 32
// lanes in turn in the host emulation, so lane layouts, MMA fragments and shuffles are checked on the CPU too.
// Per-lane values are arrays [WB_CL] indexed by WB_LI(lane).
#ifdef WB_EMU
#define WB_CL 32
#define WB_FOR_LANES(l) for (int l = 0; l < 32; ++l)
#else
#define WB_CL 1
#define WB_FOR_LANES(l) for (int l = (int)(threadIdx.x & 31), wb_once_ = 1; wb_once_; wb_once_ = 0)
#endif
#define WB_LI(l) ((WB_CL == 1) ? 0 : (l))

namespace wb {

#ifndef WB_EMU
// D = A B + D, one m16n8k8 FP64 tensor-core MMA (DMMA).  Fragments of lane (g, t) = (lane / 4, lane % 4): a0 / a1 =
// A[g][t] / A[g + 8][t], a2 / a3 = A[g][t + 4] / A[g + 8][t + 4]; b0 / b1 = B[t][g] / B[t + 4][g]; d0, d1 = D[g][2t],
// D[g][2t + 1]; d2, d3 = D[g + 8][2t], D[g + 8][2t + 1].
WB_DEV void mma_f64_16x8x8(double (&d)[4], double a0, double a1, double a2, double a3, double b0, double b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
}
#endif

// The same MMA on lane-generic fragments: a[lane] = {a0, a1, a2, a3}, b[lane] = {b0, b1}, d[lane] = {d0, d1, d2, d3}.
// The host emulation assembles A and B from all 32 lanes' fragments and accumulates each D[r][c] with fma in k order.
WB_DEV void mma_f64_16x8x8(double (&d)[WB_CL][4], const double (&a)[WB_CL][4], const double (&b)[WB_CL][2]) {
#ifdef WB_EMU
  double A[16][8], B[8][8];
  for (int l = 0; l < 32; ++l) {
    const int g = l >> 2, t = l & 3;
    A[g][t] = a[l][0]; A[g + 8][t] = a[l][1]; A[g][t + 4] = a[l][2]; A[g + 8][t + 4] = a[l][3];
    B[t][g] = b[l][0]; B[t + 4][g] = b[l][1];
  }
  for (int l = 0; l < 32; ++l) {
    const int g = l >> 2, t = l & 3;
    for (int e = 0; e < 4; ++e) {
      const int r = g + 8 * (e >> 1), c = 2 * t + (e & 1);
      double acc = d[l][e];
      for (int k = 0; k < 8; ++k) acc = fma(A[r][k], B[k][c], acc);
      d[l][e] = acc;
    }
  }
#else
  mma_f64_16x8x8(d[0], a[0][0], a[0][1], a[0][2], a[0][3], b[0][0], b[0][1]);
#endif
}

}  // namespace wb
