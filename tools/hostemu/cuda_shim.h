// Host emulation shim: lets g++ compile the kernel templates of kornia_b200/csrc/*.cuh as plain C++ so that
// tools/hostemu/run_emu.cpp can EXECUTE them on the CPU, one fiber per CUDA thread (see hostemu.h, README.md).
// Force-included before every other header:  g++ -include tools/hostemu/cuda_shim.h ...
// Nothing here is used by the product build (nvcc never sees KB200_HOST_EMU).
#pragma once
#define KB200_HOST_EMU 1
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

// CUDA keywords -> nothing (host_defines.h maps them to attributes gcc does not know)
#undef __global__
#undef __device__
#undef __host__
#undef __shared__
#undef __forceinline__
#undef __noinline__
#undef __launch_bounds__
#undef __grid_constant__
#undef __align__
#define __global__
#define __device__
#define __host__
#define __shared__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __grid_constant__
#define __align__(n) __attribute__((aligned(n)))

// built-in variables: set by the fiber scheduler before a fiber runs
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;

using std::max;
using std::min;

// ---- block-level primitives implemented by the scheduler (hostemu.h)
void __syncthreads();
int __syncthreads_or(int pred);

// ---- arithmetic intrinsics: compile with -ffp-contract=off so that plain a * b + c is never fused
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline double __fma_rn(double a, double b, double c) { return fma(a, b, c); }
inline float __double2float_rn(double a) { return (float)a; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline double __dsqrt_rn(double a) { return sqrt(a); }
inline float2 __ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
inline int __float_as_int(float f) {
  int i;
  memcpy(&i, &f, 4);
  return i;
}
inline float __int_as_float(int i) {
  float f;
  memcpy(&f, &i, 4);
  return f;
}
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline float __uint_as_float(unsigned u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// PRMT in its default mode: result byte i = byte (selector nibble i) of the 8-byte pool {x: 0..3, y: 4..7}
inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
  const unsigned long long pool = ((unsigned long long)y << 32) | x;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((pool >> (8 * ((s >> (4 * i)) & 7))) & 255) << (8 * i);
  return r;
}
template <typename T>
inline T __ldg(const T* p) { return *p; }
template <typename T>
inline void __stcs(T* p, T v) { *p = v; }
inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
inline size_t __cvta_generic_to_global(const void* p) { return (size_t)p; }

// ---- warp-level intrinsics: rendezvous of the 32 fibers of a warp (hostemu.h).  Every lane of the warp must reach
// the same sequence of collectives (converged code with the full mask, which is how the kernels use them).
float __fadd_rd(float, float);
unsigned __ballot_sync(unsigned, int);
int __all_sync(unsigned, int);
int __any_sync(unsigned, int);
void __syncwarp(unsigned = 0xffffffffu);
unsigned long long emu_warp_exchange(unsigned long long mine, int src_lane);  // deposit, rendezvous, read src_lane's deposit
int emu_lane();
template <typename T>
inline T __shfl_xor_sync(unsigned, T v, int o, int = 32) {
  static_assert(sizeof(T) <= 8, "shuffle payload");
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  bits = emu_warp_exchange(bits, emu_lane() ^ o);
  memcpy(&v, &bits, sizeof(T));
  return v;
}
template <typename T>
inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32) {
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  const int lane = emu_lane();
  bits = emu_warp_exchange(bits, lane >= (int)d ? lane - (int)d : lane);
  memcpy(&v, &bits, sizeof(T));
  return v;
}
template <typename T>
inline T __shfl_sync(unsigned, T v, int src, int = 32) {
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  bits = emu_warp_exchange(bits, src);
  memcpy(&v, &bits, sizeof(T));
  return v;
}
int atomicAdd(int*, int);
float atomicAdd(float*, float);
double atomicAdd(double*, double);
int atomicMax(int*, int);
inline int __ffs(int x) { return __builtin_ffs(x); }
