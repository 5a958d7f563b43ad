// kornia_b200 -- PatchDominantGradientOrientation.forward as one kernel: Sobel gradients, an A-bin orientation histogram
// per patch (the mean over the patch of each bin's one-hot weights), the circular 5-tap smoothing, the first maximal
// bin (NaN wins, as torch.max) and the parabolic sub-bin offset.  Staging, binning and the fixed-order sums are those of
// patch_hist.cuh; warp w sums the bins w, w + 8, ... with each lane taking every 32nd pixel in order, then a butterfly.
#pragma once
#include "patch_hist.cuh"

namespace kb200 {

struct OriParams {
  const float* src;
  const float* weighting;  // P x P Gaussian weighting (the module's weighting)
  const float* smooth;     // 5 taps (the module's angular_smooth.weight)
  float* out;              // N angles
  long long sB, sH;
  long long N;
  int P, A;
  float eps;
};

__host__ __device__ inline int ori_smem_floats(int P, int A) { return 4 * P * P + 2 * A; }

__global__ void __launch_bounds__(PH_NT) patch_orientation_kernel(const OriParams p) {
  extern __shared__ __align__(128) unsigned char ori_smem[];
  const int P = p.P, PP = P * P, A = p.A;
  float* s_patch = reinterpret_cast<float*>(ori_smem);
  float* s_w0 = s_patch + PP;
  float* s_w1 = s_w0 + PP;
  int* s_b0 = reinterpret_cast<int*>(s_w1 + PP);
  float* s_hist = reinterpret_cast<float*>(s_b0 + PP);
  float* s_smooth = s_hist + A;
  const GradStencil st = sobel_stencil();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double count = (double)PP;
  for (long long n = blockIdx.x; n < p.N; n += gridDim.x) {
    ph_stage(p.src, p.sB, p.sH, n, P, s_patch);
    __syncthreads();
    for (int e = threadIdx.x; e < PP; e += PH_NT) {
      int b0;
      float w0, w1;
      ph_bin_pixel<true>(s_patch, P, e, st, p.eps, ldg(p.weighting + e), A, b0, w0, w1);
      s_b0[e] = b0;
      s_w0[e] = w0;
      s_w1[e] = w1;
    }
    __syncthreads();
    for (int i = warp; i < A; i += PH_NW) {
      double acc = 0.0;  // fp64, rounded once: see patch_hist.cuh
      for (int e = lane; e < PP; e += 32) acc += (double)ph_bin_value(s_b0[e], s_w0[e], s_w1[e], i, A);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) s_hist[i] = __double2float_rn(acc / count);  // adaptive_avg_pool2d to 1 x 1: the mean
    }
    __syncthreads();
    // circular 5-tap cross-correlation: out[i] = sum_k w[k] * h[(i + k - 2) mod A]
    for (int i = threadIdx.x; i < A; i += PH_NT) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        int j = (i + k - 2) % A;
        j = j < 0 ? j + A : j;
        acc = __fmaf_rn(ldg(p.smooth + k), s_hist[j], acc);
      }
      s_smooth[i] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int idx = 0;
      float c = s_smooth[0];
      for (int i = 1; i < A && c == c; ++i) {
        const float v = s_smooth[i];
        if (v > c || v != v) {
          c = v;
          idx = i;
        }
      }
      const float l = s_smooth[(A + idx - 1) % A], r = s_smooth[(idx + 1) % A];
      const float c_subpix = __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(l, r)), __fsub_rn(__fadd_rn(l, r), __fmul_rn(2.f, c)));
      const float q = __fdiv_rn(__fmul_rn(PH_TWO_PI, __fadd_rn((float)idx, c_subpix)), (float)A);
      p.out[n] = -__fsub_rn(q, PH_PI);
    }
    __syncthreads();  // s_patch, s_hist and s_smooth are reused by the next patch
  }
}

int patch_orientation_forward(const float* x, const float* weighting, const float* smooth, float* out, long long N, int P, long long sB,
                              long long sH, int A, float eps, cudaStream_t st);

}  // namespace kb200
