// kornia_b200 -- the per-keypoint pyramid level and affine map of extract_patches_from_pyramid (feature/laf.py), shared by
// the patch extraction kernel (laf_patches.cuh) and the LAF affine shape kernel (affine_shape.cuh).  The op order is
// documented in laf_patches.cuh.
#pragma once
#include "sampler.cuh"

namespace kb200 {

constexpr int LP_MAX_LEVELS = 32;

// A level the kernel samples: (B_l, C, h, w) fp32 with column stride 1.
struct LevelDesc {
  const float* p;
  long long sB, sC;
  int h, w, sH;
};

// ATen's .long() of a NaN level on the device: the same conversion instruction ATen's CUDA copy kernel issues.
__device__ __forceinline__ long long level_of(float l) { return (long long)l; }

// The per-patch scalars: the chosen level (-1 when it is not one of the n_levels sampled) and the level's affine map.
struct PatchMap {
  int level;
  float t00, t01, t02, t10, t11, t12;
  float inv_w, inv_h;  // fp32 1 / (w_l - 1), 1 / (h_l - 1)
};

// The map of the LAF [[a, b, x], [c, d, y]] (pixels).  P holds the level table (lv, n_levels, max_clamp), the patch size PS,
// the normalize / select_level flags and normalize_laf's level-0 coefficients n_lin, n_tx, n_ty.
template <typename P>
__device__ __forceinline__ PatchMap laf_patch_map(const P& p, float a, float b, float x, float c, float d, float y) {
  using R = RN<float>;
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

// Host: fill p's level table (lv, n_levels, max_clamp) from n_levels pointers and 5 dims per level (h, w, batch, channel and
// row strides), and, with `normalize`, normalize_laf's level-0 coefficients.  Each level must be the halving of the one before.
template <typename P>
inline int laf_level_table(P& p, const void* const* levels, const long long* level_dims, int n_levels, int PS, bool normalize) {
  KB_CHECK_ARG(levels && level_dims, "null level table");
  for (int l = 0; l < n_levels; ++l) {
    const long long* d = level_dims + 5 * l;
    const long long h = d[0], w = d[1], sH = d[4];
    KB_CHECK_ARG(h >= 1 && w >= 1 && sH >= w && levels[l], "bad level %d: %lld x %lld, row stride %lld", l, h, w, sH);
    KB_CHECK_ARG(l == 0 || (h == level_dims[5 * (l - 1)] / 2 && w == level_dims[5 * (l - 1) + 1] / 2),
                 "level %d (%lld x %lld) is not the halving of level %d", l, h, w, l - 1);
    if ((h - 1) * sH + w > 0x7fffffffLL) {  // the sampler's tap offsets are 32-bit within a plane
      set_error("level %d plane (%lld rows of stride %lld) exceeds 2^31 elements", l, h, sH);
      return KB200_EUNSUPPORTED;
    }
    p.lv[l] = LevelDesc{(const float*)levels[l], d[2], d[3], (int)h, (int)w, (int)sH};
  }
  const int h0 = p.lv[0].h, w0 = p.lv[0].w;
  if (normalize) {
    KB_CHECK_ARG(h0 > 1 && w0 > 1, "normalising LAFs needs an image of at least 2 x 2, got %d x %d", h0, w0);
    // normalize_laf: fp32 ones / min_size, and the Python doubles 1 / (w - 1), 1 / (h - 1) rounded to fp32
    p.n_lin = 1.0f / (float)(h0 - 1 < w0 - 1 ? h0 - 1 : w0 - 1);
    p.n_tx = (float)(1.0 / (double)(w0 - 1));
    p.n_ty = (float)(1.0 / (double)(h0 - 1));
  }
  const int max_level = (h0 < w0 ? h0 : w0) / PS;
  p.max_clamp = (float)(max_level - 1 > 0 ? max_level - 1 : 0);
  p.n_levels = n_levels;
  return KB200_OK;
}

}  // namespace kb200
