// kornia_b200 -- SIFTDescriptor.forward as one kernel: per-pixel binning (patch_hist.cuh), then each of the
// A * S * S pooled cells summed by one owner thread over its K x K window, and the fixed-order L2 / clamp / L2 / RootSIFT
// normalisation.
#pragma once
#include "patch_hist.cuh"

namespace kb200 {

struct SiftParams {
  const float* src;
  const float* gk;  // P x P Gaussian weighting (the module's gk)
  const float* pk;  // K x K pooling weights (the module's pk.weight)
  float* out;       // N x D, D = A * S * S
  long long sB, sH;
  long long N;
  int P, A, S, K, stride, pad;
  int rootsift;
  float clipval, eps;
};

__host__ __device__ inline int sift_smem_floats(int P, int K, int D) { return 2 * PH_NW + 4 * P * P + K * K + D; }

__global__ void __launch_bounds__(PH_NT) sift_describe_kernel(const SiftParams p) {
  extern __shared__ __align__(128) unsigned char sift_smem[];
  const int P = p.P, PP = P * P, A = p.A, S = p.S, K = p.K, D = A * S * S;
  double* s_red = reinterpret_cast<double*>(sift_smem);
  float* s_patch = reinterpret_cast<float*>(s_red + PH_NW);
  float* s_w0 = s_patch + PP;
  float* s_w1 = s_w0 + PP;
  int* s_b0 = reinterpret_cast<int*>(s_w1 + PP);
  float* s_pk = reinterpret_cast<float*>(s_b0 + PP);
  float* s_desc = s_pk + K * K;
  for (int e = threadIdx.x; e < K * K; e += PH_NT) s_pk[e] = ldg(p.pk + e);
  const GradStencil st = diff_stencil();
  for (long long n = blockIdx.x; n < p.N; n += gridDim.x) {
    ph_stage(p.src, p.sB, p.sH, n, P, s_patch);
    __syncthreads();
    for (int e = threadIdx.x; e < PP; e += PH_NT) {
      int b0;
      float w0, w1;
      ph_bin_pixel<false>(s_patch, P, e, st, p.eps, ldg(p.gk + e), A, b0, w0, w1);
      s_b0[e] = b0;
      s_w0[e] = w0;
      s_w1[e] = w1;
    }
    __syncthreads();
    // pooled cell c = (i, sy, sx): the strided zero-padded K x K window of angular plane i, taps in row-major order
    // (a padded tap adds w * 0, as the convolution over a zero-padded plane does)
    double part = 0.0;
    for (int c = threadIdx.x; c < D; c += PH_NT) {
      const int i = c / (S * S), cell = c - i * S * S, sy = cell / S, sx = cell - sy * S;
      const int y0 = sy * p.stride - p.pad, x0 = sx * p.stride - p.pad;
      double acc = 0.0;
      for (int ky = 0; ky < K; ++ky) {
        const int y = y0 + ky;
        const bool yin = (unsigned)y < (unsigned)P;
        for (int kx = 0; kx < K; ++kx) {
          const int x = x0 + kx;
          float v = 0.f;
          if (yin && (unsigned)x < (unsigned)P) {
            const int e = y * P + x;
            v = ph_bin_value(s_b0[e], s_w0[e], s_w1[e], i, A);
          }
          acc = __fma_rn((double)s_pk[ky * K + kx], (double)v, acc);
        }
      }
      const float cell_sum = __double2float_rn(acc);
      s_desc[c] = cell_sum;
      part = __fma_rn((double)cell_sum, (double)cell_sum, part);
    }
    // L2-normalise, clamp to [0, clipval], L2-normalise; RootSIFT: sqrt(L1-normalise + eps)
    float div = ph_norm_divisor(__double2float_rn(sqrt(ph_block_sum(part, s_red))));
    part = 0.0;
    for (int c = threadIdx.x; c < D; c += PH_NT) {
      float v = __fdiv_rn(s_desc[c], div);
      if (v == v) v = fminf(fmaxf(v, 0.f), p.clipval);
      s_desc[c] = v;
      part = __fma_rn((double)v, (double)v, part);
    }
    div = ph_norm_divisor(__double2float_rn(sqrt(ph_block_sum(part, s_red))));
    float* out = p.out + n * D;
    if (p.rootsift) {
      part = 0.0;
      for (int c = threadIdx.x; c < D; c += PH_NT) {
        const float v = __fdiv_rn(s_desc[c], div);
        s_desc[c] = v;
        part += fabs((double)v);
      }
      div = ph_norm_divisor(__double2float_rn(ph_block_sum(part, s_red)));
      for (int c = threadIdx.x; c < D; c += PH_NT) out[c] = __fsqrt_rn(__fadd_rn(__fdiv_rn(s_desc[c], div), p.eps));
    } else {
      for (int c = threadIdx.x; c < D; c += PH_NT) out[c] = __fdiv_rn(s_desc[c], div);
    }
    __syncthreads();  // s_patch, s_desc and s_red are reused by the next patch
  }
}

int sift_describe_forward(const float* x, const float* gk, const float* pk, float* out, long long N, int P, long long sB, long long sH, int A,
                          int S, int K, int stride, int pad, int rootsift, float clipval, float eps, cudaStream_t st);

}  // namespace kb200
