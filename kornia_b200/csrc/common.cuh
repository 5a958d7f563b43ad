// kornia_b200 -- shared device/host helpers (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/kornia_b200.h"

namespace kb200 {

// ---------------------------------------------------------------- error plumbing (capi.cu)
void set_error(const char* fmt, ...);

#define KB_CHECK_ARG(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      ::kb200::set_error(__VA_ARGS__);   \
      return KB200_EINVAL;               \
    }                                    \
  } while (0)

#define KB_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess) {                                                                 \
      ::kb200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return KB200_ECUDA;                                                                     \
    }                                                                                         \
  } while (0)

// ---------------------------------------------------------------- separately rounded arithmetic
// The eager reference evaluates the coordinate chain as one torch kernel per op, so every
// product / sum is rounded on its own (no FMA contraction).  The _rn intrinsics are never
// contracted by nvcc, which keeps the chain bit-faithful (SURVEY.md appendix A).
template <typename T>
struct RN;

template <>
struct RN<float> {
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
  static __device__ __forceinline__ float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
  static __device__ __forceinline__ float floor(float a) { return floorf(a); }
  static __device__ __forceinline__ float rint(float a) { return rintf(a); }
  static __device__ __forceinline__ float abs(float a) { return fabsf(a); }
  static __device__ __forceinline__ float fmod(float a, float b) { return fmodf(a, b); }
};

template <>
struct RN<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
  static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
  static __device__ __forceinline__ double floor(double a) { return ::floor(a); }
  static __device__ __forceinline__ double rint(double a) { return ::rint(a); }
  static __device__ __forceinline__ double abs(double a) { return ::fabs(a); }
  static __device__ __forceinline__ double fmod(double a, double b) { return ::fmod(a, b); }
};

// read-only, L1-allocating global load (gathers reuse neighbouring taps through L1)
template <typename T>
__device__ __forceinline__ T ldg(const T* p) {
  return __ldg(p);
}

// streaming store: the output is written once and never re-read by this kernel
__device__ __forceinline__ void st_stream(float* p, float v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream(double* p, double v) { __stcs(p, v); }

__host__ __device__ __forceinline__ int ceil_div(int a, int b) { return (a + b - 1) / b; }

// two fp32 FMAs on a pair of columns, each rounded once (sm_90 has no packed fp32 FMA: two FFMA per pair)
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// ---------------------------------------------------------------- kernel-selection switches (capi.cu)
// Which of the library's own kernels serves a request.  Every switch is read from the environment ONCE, when the library is
// loaded (KB200_<NAME>=0|1), and can be changed afterwards through kb200_set_option (tests compare a tiled kernel with the
// kernel it stands in for): no getenv on the call path.
enum Option {
  OPT_TMA,             // TMA-tiled warp / remap / backward kernels (off: the generic per-pixel kernels)
  OPT_TILED_FILTER,    // shared-memory filter kernels (off: filter_generic.cuh)
  OPT_SQUARE_TILES,    // second tile shape of the forward warp for rotated samples
  OPT_TILED_GRADIENT,  // shared-memory derivative stencils (off: gradient.cuh)
  OPT_U8_TILED,        // staged-window uint8 ingest warp (off: per-tap kernel)
  OPT_BWD_STRIDE1,     // tiled backward on stride-1 lanes (default; 0: the column-pair lanes, dealt out in advance).  At cfg4
                       // the column pairs were 5 % slower on a B200; on an H100 SXM at 400 W, one alternated A/B had them
                       // 2.6 % faster (4.69 vs 4.81 ms per launch).  On an H100 SXM at 700 W, 4 alternated runs each of
                       // bench.py --workload warp_bwd (kernel ms, median): default 4.78, bwd_stride1=0 4.66, dyn_sched=0
                       // (stride-1 lanes, static deal) 4.63: the default's deficit is the run-time deal's, not the lanes'.
  OPT_DYN_SCHED,       // warp forward and backward: work handed out at run time (off: dealt out in advance)
  OPT_COUNT
};
int option(Option o);

// cudaFuncSetAttribute is per device: remember, per kernel instantiation, on which devices it was applied.  The bit is set
// only AFTER the attribute call returned (see KB_SET_SMEM_ONCE), and atomically: two host threads driving different GPUs
// (ctypes releases the GIL) may both apply the attribute, never launch without it.
inline bool needs_attribute_on_device(const unsigned long long& mask, int& dev) {
  dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return true;
  return (__atomic_load_n(&mask, __ATOMIC_ACQUIRE) & (1ull << (dev & 63))) == 0;
}
inline void attribute_applied_on_device(unsigned long long& mask, int dev) { __atomic_fetch_or(&mask, 1ull << (dev & 63), __ATOMIC_RELEASE); }

// Work counters of the run-time work distribution: a ring of 1 024 counters per device, allocated once (128 KB, the library's only
// device allocation), one slot per launch, zeroed on the launch's stream.  A slot comes round again after 1 024 launches; two
// launches could only share one if the first were still running then.  (A counter taken from the default memory pool with
// cudaMallocAsync / cudaFreeAsync around each launch made whole runs of the headline bench markedly slower than others.)
inline int* take_work_counter(cudaStream_t st) {
  constexpr int SLOTS = 1024, STRIDE = 32;  // ints: one counter per 128-byte line
  static int* base[64] = {nullptr};
  static unsigned long long seq[64] = {0};
  static int lock = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  int* b = __atomic_load_n(&base[dev], __ATOMIC_ACQUIRE);
  if (!b) {
    while (__atomic_exchange_n(&lock, 1, __ATOMIC_ACQUIRE)) {
    }
    b = base[dev];
    if (!b) {
      void* ptr = nullptr;
      if (cudaMalloc(&ptr, (size_t)SLOTS * STRIDE * sizeof(int)) == cudaSuccess) {
        b = static_cast<int*>(ptr);
        __atomic_store_n(&base[dev], b, __ATOMIC_RELEASE);
      } else {
        (void)cudaGetLastError();
      }
    }
    __atomic_store_n(&lock, 0, __ATOMIC_RELEASE);
    if (!b) return nullptr;
  }
  int* slot = b + (size_t)(__atomic_fetch_add(&seq[dev], 1ull, __ATOMIC_RELAXED) % SLOTS) * STRIDE;
  if (cudaMemsetAsync(slot, 0, sizeof(int), st) != cudaSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  return slot;
}

#define KB_SET_SMEM_ONCE(mask, kern, bytes)                                                                   \
  do {                                                                                                       \
    int dev__ = 0;                                                                                           \
    if (::kb200::needs_attribute_on_device(mask, dev__)) {                                                   \
      KB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));        \
      ::kb200::attribute_applied_on_device(mask, dev__);                                                     \
    }                                                                                                        \
  } while (0)

}  // namespace kb200
