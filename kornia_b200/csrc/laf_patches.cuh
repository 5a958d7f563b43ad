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
#include "sampler.cuh"

namespace kb200 {

constexpr int LP_NT = 128;          // threads per CTA: 19 x 19 = 361 pixels are 3 rounds of 128 (94 % of the lanes busy)
constexpr int LP_MAX_LEVELS = 32;

// A level the kernel samples: (B_l, C, h, w) fp32 with column stride 1.
struct LevelDesc {
  const float* p;
  long long sB, sC;
  int h, w, sH;
};

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

// ATen's .long() of a NaN level on the device: the same conversion instruction ATen's CUDA copy kernel issues.
__device__ __forceinline__ long long level_of(float l) { return (long long)l; }

// The per-patch scalars: the chosen level (-1 when it is not one of the n_levels sampled) and the level's affine map.
struct PatchMap {
  int level;
  float t00, t01, t02, t10, t11, t12;
  float inv_w, inv_h;  // fp32 1 / (w_l - 1), 1 / (h_l - 1)
};

__device__ __forceinline__ PatchMap laf_patch_map(const LafPatchParams& p, long long n) {
  using R = RN<float>;
  const float* L = p.laf + n * 6;
  float a = ldg(L + 0), b = ldg(L + 1), x = ldg(L + 2), c = ldg(L + 3), d = ldg(L + 4), y = ldg(L + 5);
  if (p.normalize) {
    a = R::mul(p.n_lin, a); b = R::mul(p.n_lin, b); x = R::mul(p.n_tx, x);
    c = R::mul(p.n_lin, c); d = R::mul(p.n_lin, d); y = R::mul(p.n_ty, y);
  }
  PatchMap m;
  int lvl = 0;
  if (p.select_level) {
    const float m0 = (float)min(p.lv[0].h - 1, p.lv[0].w - 1);
    const float da = R::mul(m0, a), db = R::mul(m0, b), dc = R::mul(m0, c), dd = R::mul(m0, d);
    const float det = R::add(R::sub(R::mul(da, dd), R::mul(dc, db)), 1e-10f);
    const float s = R::mul(R::mul(2.0f, __fsqrt_rn(fabsf(det))), R::div(1.0f, (float)p.PS));
    float l = log2f(s);
    if (!(l != l)) l = fminf(fmaxf(l, 0.0f), p.max_clamp);
    const long long L64 = level_of(l);
    lvl = (L64 >= 0 && L64 < p.n_levels) ? (int)L64 : -1;
  }
  m.level = lvl;
  if (lvl < 0) return m;
  const int h = p.lv[lvl].h, w = p.lv[lvl].w;
  const float ml = (float)min(h - 1, w - 1), wf = (float)(w - 1), hf = (float)(h - 1);
  m.t00 = R::mul(ml, a); m.t01 = R::mul(ml, b); m.t02 = R::mul(wf, x);
  m.t10 = R::mul(ml, c); m.t11 = R::mul(ml, d); m.t12 = R::mul(hf, y);
  m.inv_w = R::div(1.0f, wf);
  m.inv_h = R::div(1.0f, hf);
  return m;
}

// The normalised sampling coordinate of base point (bx, by) (grid_sample's input, before unnormalize).
__device__ __forceinline__ void laf_grid_point(const PatchMap& m, float bx, float by, float& gx, float& gy) {
  using R = RN<float>;
  gx = R::add(R::fma(by, m.t01, R::mul(bx, m.t00)), m.t02);
  gy = R::add(R::fma(by, m.t11, R::mul(bx, m.t10)), m.t12);
  gx = R::sub(R::mul(R::mul(2.0f, gx), m.inv_w), 1.0f);
  gy = R::sub(R::mul(R::mul(2.0f, gy), m.inv_h), 1.0f);
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
