// kornia_b200 -- PatchAffineShapeEstimator.forward and LAFAffineShapeEstimator.forward (feature/affine_shape.py), each as
// one kernel: one CTA per keypoint (persistent CTAs), the patch in shared memory, the Baumberg second-moment matrix of its
// weighted Sobel gradients, then a scalar tail on thread 0.
//
// Moments (both kernels), per pixel in the reference's fp32 op order, no contraction:
//   (gx, gy) = the sobel_stencil() gradient over a replicate border (spatial_gradient's arithmetic, patch_hist.cuh)
//   gx *= weighting, gy *= weighting  (grads * weighting: the weighting multiplies the gradients before they are squared)
//   gx * gx, gx * gy, gy * gy          (pow(2) is a product)
// Each product is summed in fp64 in a fixed order (per thread, then ph_block_sum), divided by P^2 and rounded once.  The
// reference's two fp32 means are pairwise sums; fp64 makes the kernel's moments the correctly rounded ones.
// Tail: degenerate when at least two of (a, b, c) are < eps (a negative b counts); shape * (1 - bad) + [1, 0, 1] * bad as
// fp32 products and an add (so a NaN moment stays NaN); divided by the first maximal element, NaN winning as in torch.max.
//
// LAF kernel, per keypoint [[a, b, x], [c, d, y]]:
//   make_upright:   det = sqrt(|a d - c b + 1e-10|), b2a2 = sqrt(b^2 + a^2) + 1e-9,
//                   U = det * [[b2a2 / det, 0], [(d b + c a) / (b2a2 det), det / b2a2]]
//   the patch:      laf_patch_map / laf_grid_point (laf_map.cuh) of U and PixelSampler<BILINEAR, BORDER>, straight into shared
//                   memory; a keypoint whose level is not among those sampled has a zero patch (the circular shape)
//   ellipse_to_laf: a11 = sqrt|A|, a22 = sqrt|C|, a21 = B / max(a11 + a22, 1e-9) (NaN propagating, as clamp); the inverse of
//                   the lower-triangular [[a11, 0], [a21, a22]] in closed form: [[1 / a11, 0], [-(a21 / (a11 a22)), 1 / a22]]
//                   (torch.inverse's LU may differ by ulps, and leave an ulp-sized upper-right entry)
//   rescale:        * (det / get_laf_scale(out))
//   orientation:    (preserve_orientation) rotate by rad2deg(atan2(b, a)) - rad2deg(atan2(o01, o00)) degrees: deg2rad as on
//                   the device ((v * pi) * fp32(1 / 180)), [[cos, sin], [-sin, cos]], the 2 x 2 product as fma(l1, r1, l0 * r0)
//   centre:         copied from the input.
#pragma once
#include "laf_map.cuh"
#include "patch_hist.cuh"

namespace kb200 {

struct PatchAffParams {
  const float* src;        // (N, 1, P, P), column stride 1
  const float* weighting;  // P x P
  float* out;              // (N, 3)
  long long sB, sH, N;
  int P;
  float eps;
};

struct LafAffParams {
  LevelDesc lv[LP_MAX_LEVELS];
  const float* laf;        // (B, N, 2, 3) contiguous
  const float* base;       // PS base-grid coordinates of affine_grid(align_corners=False)
  const float* weighting;  // PS x PS
  float* out;              // (B, N, 2, 3) contiguous
  long long N, total;
  int PS, n_levels;
  float n_lin, n_tx, n_ty, max_clamp;
  float eps;
  int preserve_orientation;
  static constexpr int normalize = 1, select_level = 1;  // extract_patches_from_pyramid(img, make_upright(laf), PS, True)
};

// The three moments of the staged P x P patch; every thread returns them.  `red` holds PH_NW doubles.
__device__ __forceinline__ void aff_moments(const float* s_patch, int P, const float* __restrict__ weighting, double* red, float m[3]) {
  const GradStencil st = sobel_stencil();
  double s[3] = {0.0, 0.0, 0.0};
  for (int e = threadIdx.x; e < P * P; e += PH_NT) {
    float g[2];
    ph_gradient(s_patch, P, e, st, g);
    const float w = ldg(weighting + e);
    const float gx = __fmul_rn(g[0], w), gy = __fmul_rn(g[1], w);
    s[0] += (double)__fmul_rn(gx, gx);
    s[1] += (double)__fmul_rn(gx, gy);
    s[2] += (double)__fmul_rn(gy, gy);
  }
  const double count = (double)(P * P);
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = __double2float_rn(ph_block_sum(s[k], red) / count);
}

// PatchAffineShapeEstimator's tail: the degenerate mask, the circular replacement and the max normalisation.
__device__ __forceinline__ void aff_shape_tail(float m[3], float eps) {
  const float bad = ((m[0] < eps) + (m[1] < eps) + (m[2] < eps)) >= 2 ? 1.f : 0.f;
  const float keep = __fsub_rn(1.f, bad);
  const float circ[3] = {1.f, 0.f, 1.f};
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = __fadd_rn(__fmul_rn(m[k], keep), __fmul_rn(circ[k], bad));
  float mx = m[0];
#pragma unroll
  for (int k = 1; k < 3; ++k)
    if (m[k] > mx || m[k] != m[k]) mx = m[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = __fdiv_rn(m[k], mx);
}

// get_laf_scale of [[a, b], [c, d]]: sqrt(|a d - c b + 1e-10|).
__device__ __forceinline__ float aff_laf_scale(float a, float b, float c, float d) {
  return __fsqrt_rn(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(a, d), __fmul_rn(c, b)), 1e-10f)));
}

// rad2deg(atan2(y, x)): 180 * t / pi, pi the fp32 constant.
__device__ __forceinline__ float aff_angle_deg(float y, float x) { return __fdiv_rn(__fmul_rn(180.f, atan2f(y, x)), PH_PI); }

// The LAF tail from the normalised shape m and the input LAF's linear part (a, b, c, d) with its scale det: writes the
// linear part of the output LAF to o[0..3] (row-major).
__device__ __forceinline__ void aff_laf_tail(const float m[3], float a, float b, float det, bool preserve, float o[4]) {
  using R = RN<float>;
  const float a11 = __fsqrt_rn(fabsf(m[0])), a22 = __fsqrt_rn(fabsf(m[2]));
  float den = R::add(a11, a22);
  den = den != den ? den : fmaxf(den, 1e-9f);
  const float a21 = R::div(m[1], den);
  const float i00 = R::div(1.f, a11), i11 = R::div(1.f, a22), i10 = -R::div(a21, R::mul(a11, a22)), i01 = 0.f;
  const float coef = R::div(det, aff_laf_scale(i00, i01, i10, i11));
  o[0] = R::mul(coef, i00);
  o[1] = R::mul(coef, i01);
  o[2] = R::mul(coef, i10);
  o[3] = R::mul(coef, i11);
  if (!preserve) return;
  const float ang = R::sub(aff_angle_deg(b, a), aff_angle_deg(o[1], o[0]));
  const float rad = R::mul(R::mul(ang, PH_PI), R::div(1.f, 180.f));
  const float cs = cosf(rad), sn = sinf(rad), r[2][2] = {{cs, sn}, {-sn, cs}};
  const float l[2][2] = {{o[0], o[1]}, {o[2], o[3]}};
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) o[2 * i + j] = R::fma(l[i][1], r[1][j], R::mul(l[i][0], r[0][j]));
}

__global__ void __launch_bounds__(PH_NT) patch_affine_shape_kernel(const PatchAffParams p) {
  extern __shared__ __align__(128) unsigned char paff_smem[];
  double* s_red = reinterpret_cast<double*>(paff_smem);
  float* s_patch = reinterpret_cast<float*>(s_red + PH_NW);
  for (long long n = blockIdx.x; n < p.N; n += gridDim.x) {
    ph_stage(p.src, p.sB, p.sH, n, p.P, s_patch);
    __syncthreads();
    float m[3];
    aff_moments(s_patch, p.P, p.weighting, s_red, m);  // its block sums end with a barrier: s_patch is free again
    if (threadIdx.x == 0) {
      aff_shape_tail(m, p.eps);
#pragma unroll
      for (int k = 0; k < 3; ++k) p.out[3 * n + k] = m[k];
    }
  }
}

__global__ void __launch_bounds__(PH_NT) laf_affine_shape_kernel(const __grid_constant__ LafAffParams p) {
  using R = RN<float>;
  extern __shared__ __align__(128) unsigned char laff_smem[];
  double* s_red = reinterpret_cast<double*>(laff_smem);
  float* s_patch = reinterpret_cast<float*>(s_red + PH_NW);
  const int PS = p.PS, PP = PS * PS;
  for (long long n = blockIdx.x; n < p.total; n += gridDim.x) {
    const float* L = p.laf + n * 6;
    const float a = ldg(L + 0), b = ldg(L + 1), x = ldg(L + 2), c = ldg(L + 3), d = ldg(L + 4), y = ldg(L + 5);
    // make_upright
    const float det = aff_laf_scale(a, b, c, d);
    const float b2a2 = R::add(__fsqrt_rn(R::add(R::mul(b, b), R::mul(a, a))), 1e-9f);
    const float u00 = R::mul(det, R::div(b2a2, det)), u01 = R::mul(det, 0.f);
    const float u10 = R::mul(det, R::div(R::add(R::mul(d, b), R::mul(c, a)), R::mul(b2a2, det)));
    const float u11 = R::mul(det, R::div(det, b2a2));
    const PatchMap mp = laf_patch_map(p, u00, u01, x, u10, u11, y);
    float m[3] = {0.f, 0.f, 0.f};  // an unsampled level: a zero patch has zero moments
    if (mp.level >= 0) {           // uniform across the CTA
      const LevelDesc& lv = p.lv[mp.level];
      const float* src = lv.p + (n / p.N) * lv.sB;
      for (int e = threadIdx.x; e < PP; e += PH_NT) {
        const int i = e / PS, j = e - i * PS;
        float gx, gy;
        laf_grid_point(mp, ldg(p.base + j), ldg(p.base + i), gx, gy);
        PixelSampler<float, KB200_BILINEAR, KB200_BORDER> ps;
        ps.prepare_rows(unnormalize(gx, lv.w, false), unnormalize(gy, lv.h, false), lv.h, lv.w, lv.sH, false);
        s_patch[e] = ps.sample(src);
      }
      __syncthreads();
      aff_moments(s_patch, PS, p.weighting, s_red, m);  // ends with a barrier: s_patch is free again
    }
    if (threadIdx.x == 0) {
      aff_shape_tail(m, p.eps);
      float o[4];
      aff_laf_tail(m, a, b, det, p.preserve_orientation, o);
      float* out = p.out + n * 6;
      out[0] = o[0];
      out[1] = o[1];
      out[2] = x;
      out[3] = o[2];
      out[4] = o[3];
      out[5] = y;
    }
  }
}

// Dynamic shared memory: the block-sum slots, then the P x P patch.
__host__ __device__ inline int aff_smem_bytes(int P) { return (int)(PH_NW * sizeof(double) + sizeof(float) * P * P); }

int patch_affine_shape_forward(const float* x, const float* weighting, float* out, long long N, int P, long long sB, long long sH, float eps,
                               cudaStream_t st);
int laf_affine_shape_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                             const void* weighting, void* out, long long B, long long N, int PS, float eps, int preserve_orientation,
                             cudaStream_t st);

}  // namespace kb200
