// wb_platform.cuh -- one place that knows whether the kernel sources are being compiled by
// nvcc for sm_90a (the product) or by g++ as a single-thread host emulation (tests only).
//
// The emulation exists because the development container has no GPU: every kernel in this
// tree is written block-size-agnostic (strided `for (i = tid; i < n; i += nthreads)` phases
// separated by barriers, warp-level tricks hidden behind the helpers in wb_block.cuh), so the
// very same source can be run with one "thread" per block on the CPU to check the arithmetic
// against the oracle before spending GPU minutes.  The emulation build lives under tests/
// (tests/emu), is never loaded by world_b200/ and is NOT a fallback: libworld_b200.so is
// CUDA-only and fails loudly without a device.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <math.h>
#include <string.h>

#ifndef WB_EMU
// ----------------------------------------------------------------------------- CUDA build
#include <cuda_runtime.h>
#define WB_HD __host__ __device__
#define WB_DEV __device__ __forceinline__
#define WB_DEV_NOINLINE static __device__ __noinline__   /* one copy per kernel: big helpers called from several places */
#define WB_DEV_MEMBER __device__ __forceinline__
#define WB_KERNEL(bounds_threads, bounds_blocks) \
  __global__ void __launch_bounds__(bounds_threads, bounds_blocks)
#define WB_KERNEL_PLAIN __global__ void
#define WB_DYN_SMEM(type, name) \
  extern __shared__ __align__(16) unsigned char wb_dyn_smem_[]; \
  type *name = reinterpret_cast<type *>(wb_dyn_smem_)
#define WB_SHARED __shared__
#define WB_SYNC() __syncthreads()
#define WB_UNROLL4  /* r1k experiment: "unroll 4" cost registers and occupancy (CheapTrick 99 -> 113 ms); kept empty */
#define WB_TID ((int)threadIdx.x)
#define WB_NTH ((int)blockDim.x)
#define WB_CONST_TABLE __device__
typedef cudaStream_t wb_stream_t;

// Cooperative kernels (block-wide phases + barriers) and flat kernels (independent threads)
// launch the same way on the device.
namespace wb {
extern unsigned long long g_launches;
extern int g_prof_on;                       // per-kernel CUDA-event timing (world_b200_profile)
void prof_begin(const char *name, cudaStream_t s);
void prof_end(cudaStream_t s);
}
#define WB_LAUNCH_COOP(kernel, grid, block, smem, stream, ...)            \
  do {                                                                    \
    ++wb::g_launches;                                                     \
    if (wb::g_prof_on) wb::prof_begin(#kernel, (stream));                 \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);           \
    if (wb::g_prof_on) wb::prof_end((stream));                            \
  } while (0)
#define WB_LAUNCH_FLAT(kernel, grid, block, smem, stream, ...) \
  WB_LAUNCH_COOP(kernel, grid, block, smem, stream, __VA_ARGS__)

#else
// ------------------------------------------------------------------- host emulation build
#include <stdlib.h>
#include <algorithm>
struct wb_dim3 {
  unsigned x, y, z;
  wb_dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
typedef wb_dim3 dim3;
extern wb_dim3 threadIdx, blockIdx, blockDim, gridDim;
extern unsigned char wb_emu_smem[];
#define WB_EMU_SMEM_BYTES (256 * 1024)
#define WB_HD
#define WB_DEV static inline
#define WB_DEV_NOINLINE static
#define WB_DEV_MEMBER inline
#define WB_KERNEL(bounds_threads, bounds_blocks) void
#define WB_KERNEL_PLAIN void
#define WB_DYN_SMEM(type, name) type *name = reinterpret_cast<type *>(wb_emu_smem)
#define WB_SHARED static
#define WB_SYNC() ((void)0)
#define WB_UNROLL4
#define WB_TID ((int)threadIdx.x)
#define WB_NTH ((int)blockDim.x)
#define WB_CONST_TABLE
#define __restrict__
typedef void *wb_stream_t;
typedef int cudaError_t;
typedef void *cudaStream_t;
#define cudaSuccess 0

namespace wb { extern unsigned long long g_launches; }
#define WB_EMU_GRID_LOOP(grid, body)                                   \
  do {                                                                 \
    wb_dim3 g_ = wb_dim3(grid);                                        \
    ++wb::g_launches;                                                  \
    gridDim = g_;                                                      \
    for (unsigned bz_ = 0; bz_ < g_.z; ++bz_)                          \
      for (unsigned by_ = 0; by_ < g_.y; ++by_)                        \
        for (unsigned bx_ = 0; bx_ < g_.x; ++bx_) {                    \
          blockIdx = wb_dim3(bx_, by_, bz_);                           \
          body                                                         \
        }                                                              \
  } while (0)

// one emulated thread per block
#define WB_LAUNCH_COOP(kernel, grid, block, smem, stream, ...)         \
  WB_EMU_GRID_LOOP(grid, {                                             \
    blockDim = wb_dim3(1, 1, 1);                                       \
    threadIdx = wb_dim3(0, 0, 0);                                      \
    kernel(__VA_ARGS__);                                               \
  })
// every thread of every block, one after the other (kernels without barriers)
#define WB_LAUNCH_FLAT(kernel, grid, block, smem, stream, ...)         \
  WB_EMU_GRID_LOOP(grid, {                                             \
    blockDim = wb_dim3(block);                                         \
    for (unsigned tx_ = 0; tx_ < blockDim.x; ++tx_) {                  \
      threadIdx = wb_dim3(tx_, 0, 0);                                  \
      kernel(__VA_ARGS__);                                             \
    }                                                                  \
  })

struct alignas(16) double2 { double x, y; };   // CUDA's double2 is 16-byte aligned: keep UBSan's alignment check meaningful
static inline double2 make_double2(double x, double y) { double2 r; r.x = x; r.y = y; return r; }
struct uint4 { unsigned x, y, z, w; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) {
  uint4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r;
}
static inline double cospi(double x) { return cos(3.1415926535897932384 * x); }   // CUDA math functions used by kernels
static inline double sinpi(double x) { return sin(3.1415926535897932384 * x); }
static inline double2 __ldg(const double2 *p) { return *p; }
static inline uint4 __ldg(const uint4 *p) { return *p; }
static inline double __ldg(const double *p) { return *p; }
static inline int __ldg(const int *p) { return *p; }
static inline unsigned __ldg(const unsigned *p) { return *p; }
#endif

// ------------------------------------------------------------------ shared small helpers
namespace wb {

// sticky per-context error word written by kernels (bit 1: window longer than fft_size,
// bit 2: smoothing width does not fit, bit 4: scratch overflow)
#ifdef WB_EMU
static inline void atomicOr_status(int *p, int v) { if (p) *p |= v; }
#else
__device__ __forceinline__ void atomicOr_status(int *p, int v) { if (p) atomicOr(p, v); }
#endif

// Arithmetic that feeds an int cast / comparison must round exactly like the reference's
// x86-64 -O1 build (no FMA).  The CUDA build is compiled with -fmad=false, so plain operators
// are already unfused; these wrappers only document intent at the call sites.
WB_HD inline double mul_rn(double a, double b) { return a * b; }
WB_HD inline double div_rn(double a, double b) { return a / b; }

// round half away from zero through an int cast (reference: matlabfunctions.cpp:206-208)
WB_HD inline int round_half_away(double x) {
  return x > 0 ? static_cast<int>(x + 0.5) : static_cast<int>(x - 0.5);
}
WB_HD inline int imin(int a, int b) { return a < b ? a : b; }
WB_HD inline int imax(int a, int b) { return a > b ? a : b; }
WB_HD inline double dmin(double a, double b) { return a < b ? a : b; }
WB_HD inline double dmax(double a, double b) { return a > b ? a : b; }

constexpr double kPi = 3.1415926535897932384;       // constantnumbers.h:18
constexpr double kTiny = 0.000000000001;            // kMySafeGuardMinimum, :19
constexpr double kEps = 0.00000000000000022204460492503131;  // :20
constexpr double kLog2 = 0.69314718055994529;       // :24

}  // namespace wb
