// kornia_b200 -- extract_patches_from_pyramid / extract_patches_simple (feature/laf.py) as one kernel: every patch's
// normalisation, scale, pyramid level and per-level affine map are computed once, then its PS x PS pixels are sampled
// bilinearly with 'border' padding (sampler.cuh, the grid_sample the reference calls) from the chosen level, every channel,
// and written once.
//
// The coordinate chain, in the reference's fp32 op order (each ATen op rounded on its own, no contraction):
//   nlaf   = laf * coef              linear part fp32 1 / min(h-1, w-1), translation the double 1/(w-1), 1/(h-1) rounded
//   scale  = (2 * sqrt(|a d - c b + 1e-10|)) * (1 / PS)   (a..d of denormalize_laf(nlaf, level 0); ATen's CUDA division by a
//                                                           Python scalar is a product with its fp32 reciprocal)
//   level  = int64(clamp(log2f(scale), 0, max_clamp))      NaN stays NaN through clamp (ATen's clamp), then converts as below
//   theta  = nlaf * coef_l            coef_l = (min(h_l-1, w_l-1), w_l-1, h_l-1) of the chosen level
//   g      = fma(by, theta_01, bx * theta_00) + theta_02   (affine_grid's bmm: the kernel fixes this order; cuBLAS's is not
//                                                           specified -- DESIGN 4.5)
//   gx     = (2 * g) * (1 / (w_l - 1)) - 1                 (likewise gy with theta_1*, h_l)
//   sample = PixelSampler<float, BILINEAR, BORDER> at unnormalize(gx, w_l), unnormalize(gy, h_l), align_corners=False
// bx, by come from the cached base vector (linspace(-1, 1, PS) * (PS - 1) / PS, built with torch ops on the device).
#pragma once
#include "laf_map.cuh"

namespace kb200 {

constexpr int LP_NT = 128;          // threads per CTA: 19 x 19 = 361 pixels are 3 rounds of 128 (94 % of the lanes busy)

struct LafPatchParams {
  LevelDesc lv[LP_MAX_LEVELS];
  const float* laf;   // (B, N, 2, 3) contiguous
  const float* base;  // PS base-grid coordinates of affine_grid(align_corners=False)
  float* out;         // (B, N, C, PS, PS) contiguous
  long long N, total;  // total = B * N patches
  int C, PS, n_levels;  // n_levels: the levels the reference samples (those built); a patch choosing another one stays zero
  int normalize, select_level;
  float n_lin, n_tx, n_ty;  // normalize_laf's coefficients for level 0
  float max_clamp;          // max(0, min(h, w) // PS - 1)
};

__device__ __forceinline__ PatchMap laf_patch_map(const LafPatchParams& p, long long n) {
  const float* L = p.laf + n * 6;
  return laf_patch_map(p, ldg(L + 0), ldg(L + 1), ldg(L + 2), ldg(L + 3), ldg(L + 4), ldg(L + 5));
}

__global__ void __launch_bounds__(LP_NT, 8) laf_patches_kernel(const __grid_constant__ LafPatchParams p) {
  const int PS = p.PS, PP = PS * PS, C = p.C;
  for (long long n = blockIdx.x; n < p.total; n += gridDim.x) {
    const PatchMap m = laf_patch_map(p, n);
    float* out = p.out + n * (long long)C * PP;
    if (m.level < 0) {
      for (long long e = threadIdx.x; e < (long long)C * PP; e += LP_NT) st_stream(out + e, 0.0f);
      continue;
    }
    const LevelDesc& L = p.lv[m.level];
    const float* src = L.p + (n / p.N) * L.sB;
    for (int e = threadIdx.x; e < PP; e += LP_NT) {
      const int i = e / PS, j = e - i * PS;
      float gx, gy;
      laf_grid_point(m, ldg(p.base + j), ldg(p.base + i), gx, gy);
      PixelSampler<float, KB200_BILINEAR, KB200_BORDER> ps;
      ps.prepare_rows(unnormalize(gx, L.w, false), unnormalize(gy, L.h, false), L.h, L.w, L.sH, false);
      for (int ch = 0; ch < C; ++ch) st_stream(out + (long long)ch * PP + e, ps.sample(src + ch * L.sC));
    }
  }
}

int extract_patches_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                            void* out, long long B, long long N, int C, int PS, int normalize, int select_level, cudaStream_t st);

}  // namespace kb200
