// kornia_b200 -- device code shared by the per-patch gradient-histogram kernels: SIFTDescriptor.forward (siftdesc.cuh)
// and PatchDominantGradientOrientation.forward (patch_orientation.cuh); the staging, gradient and block sum also serve the
// second-moment kernels of affine_shape.cuh.
//
// One CTA owns one patch at a time (persistent CTAs stride over the N patches), so a patch's result is a pure function of
// the patch: every sum runs in an order fixed by the thread layout, with no atomics and nothing depending on the grid or on
// the patch's index.
//   1. the P x P patch is staged in shared memory (batch and row strides as given, column stride 1);
//   2. each pixel's gradient (every tap of the 3 x 3 stencil, row-major FMA from 0 over a replicate border: the arithmetic
//      of spatial_gradient), magnitude, angle and angular bin are computed once, in the reference's fp32 op order with no
//      contraction, and kept as (bin, w0 = (1 - frac) * mag, w1 = frac * mag);
//   3. the histogram of angular bin i at a pixel is (b0 == i) * w0 + (b1 == i) * w1 as two real products and an add, so a
//      non-finite weight makes 0 * w = NaN in every bin, as in the reference's one-hot products;
//   4. the pooling sums and the norms accumulate in fp64 and round once to fp32: a 256-tap fp32 chain would add about
//      16 ulp of error where ATen's pairwise reductions add a few.  Each pooling tap issues three shared-memory loads for
//      one FMA, so the fp64 FMA rate is not expected to set the speed (not profiled).
#pragma once
#include "common.cuh"

namespace kb200 {

constexpr int PH_NT = 256;            // threads per CTA
constexpr int PH_NW = PH_NT / 32;
constexpr int PH_MAX_P = 64;          // patch side envelope of both kernels
constexpr int SIFT_MAX_D = 1024;      // num_ang_bins * num_spatial_bins^2
constexpr int ORI_MAX_BINS = 64;
constexpr float PH_PI = 3.14159274101257324219f;      // kornia's pi: a 0-d fp32 tensor
constexpr float PH_TWO_PI = 6.28318548202514648438f;  // 2.0 * pi, exact in fp32

// The 3 x 3 first-derivative stencils of spatial_gradient(normalized=True), [o][row][col] applied to x[y + row - 1][x + col - 1].
struct GradStencil {
  float t[2][3][3];
};
__host__ __device__ constexpr GradStencil diff_stencil() {
  return GradStencil{{{{0.f, 0.f, 0.f}, {-0.5f, 0.f, 0.5f}, {0.f, 0.f, 0.f}}, {{0.f, -0.5f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.5f, 0.f}}}};
}
__host__ __device__ constexpr GradStencil sobel_stencil() {
  return GradStencil{{{{-0.125f, 0.f, 0.125f}, {-0.25f, 0.f, 0.25f}, {-0.125f, 0.f, 0.125f}},
                      {{-0.125f, -0.25f, -0.125f}, {0.f, 0.f, 0.f}, {0.125f, 0.25f, 0.125f}}}};
}

// Stage patch n (P x P, column stride 1) into s_patch.
__device__ __forceinline__ void ph_stage(const float* __restrict__ src, long long sB, long long sH, long long n, int P, float* s_patch) {
  const float* base = src + n * sB;
  for (int e = threadIdx.x; e < P * P; e += PH_NT) {
    const int y = e / P, x = e - y * P;
    s_patch[e] = ldg(base + y * sH + x);
  }
}

// The gradient (g[0] = d/dx, g[1] = d/dy) of pixel e of the staged patch.
__device__ __forceinline__ void ph_gradient(const float* s_patch, int P, int e, const GradStencil& st, float g[2]) {
  const int y = e / P, x = e - y * P;
  g[0] = g[1] = 0.f;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int yy = min(max(y + r - 1, 0), P - 1);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = s_patch[yy * P + min(max(x + c - 1, 0), P - 1)];
#pragma unroll
      for (int o = 0; o < 2; ++o) g[o] = __fmaf_rn(st.t[o][r][c], v, g[o]);
    }
  }
}

// Pixel e of the staged patch: its first bin (-1 when the angle is NaN) and the weights of its two bins.
//   mag = sqrt(gx * gx + gy * gy + eps) * weight;  ori = atan2(gy, gx + eps) + 2 pi;  o = A * (ori [+ pi]) / (2 pi)
template <bool ADD_PI>
__device__ __forceinline__ void ph_bin_pixel(const float* s_patch, int P, int e, const GradStencil& st, float eps, float weight, int A,
                                             int& b0, float& w0, float& w1) {
  float g[2];
  ph_gradient(s_patch, P, e, st, g);
  const float gx = g[0], gy = g[1];
  float mag = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), eps));
  const float ori = __fadd_rn(atan2f(gy, __fadd_rn(gx, eps)), PH_TWO_PI);
  mag = __fmul_rn(mag, weight);
  const float o_big = __fdiv_rn(__fmul_rn((float)A, ADD_PI ? __fadd_rn(ori, PH_PI) : ori), PH_TWO_PI);
  const float f = floorf(o_big);
  const float frac = __fsub_rn(o_big, f);
  if (f != f || f - f != 0.f) {
    b0 = -1;
  } else {
    const int i = (int)f % A;  // |f| is at most 2A here; torch.remainder of an integral float
    b0 = i < 0 ? i + A : i;
  }
  w0 = __fmul_rn(__fsub_rn(1.f, frac), mag);
  w1 = __fmul_rn(frac, mag);
}

// (b0 == i) * w0 + (b1 == i) * w1 with b1 = (b0 + 1) % A, as the reference's fp32 products and add.
__device__ __forceinline__ float ph_bin_value(int b0, float w0, float w1, int i, int A) {
  const int b1 = b0 < 0 ? -1 : (b0 + 1 == A ? 0 : b0 + 1);
  return __fadd_rn(__fmul_rn(b0 == i ? 1.f : 0.f, w0), __fmul_rn(b1 == i ? 1.f : 0.f, w1));
}

// Block-wide sum of one fp64 partial per thread, in a fixed order: butterfly within each warp, then the warps in index
// order.  Every thread returns the same value.  `red` holds PH_NW doubles; the call ends with a barrier-separated read.
__device__ __forceinline__ double ph_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = red[0];
#pragma unroll
  for (int w = 1; w < PH_NW; ++w) s += red[w];
  __syncthreads();
  return s;
}

// F.normalize's divisor: max(norm, 1e-12), NaN propagating as clamp_min does.
__device__ __forceinline__ float ph_norm_divisor(float norm) { return norm < 1e-12f ? 1e-12f : norm; }

}  // namespace kb200
