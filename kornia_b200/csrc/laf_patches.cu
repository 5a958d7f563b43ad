// kornia_b200 -- host side of the LAF patch extraction kernel (laf_patches.cuh).
#include "laf_patches.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

int extract_patches_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                            void* out, long long B, long long N, int C, int PS, int normalize, int select_level, cudaStream_t st) {
  KB_CHECK_ARG(n_levels >= 1 && n_levels <= LP_MAX_LEVELS && (select_level || n_levels == 1), "bad level count %d", n_levels);
  KB_CHECK_ARG(levels && level_dims, "null level table");
  LafPatchParams p{};
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
  if (B * N == 0) return KB200_OK;
  KB_CHECK_ARG(laf && base && out, "null pointer argument");
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
  p.laf = (const float*)laf;
  p.base = (const float*)base;
  p.out = (float*)out;
  p.N = N;
  p.total = B * N;
  p.C = C;
  p.PS = PS;
  p.n_levels = n_levels;
  p.normalize = normalize;
  p.select_level = select_level;
  laf_patches_kernel<<<persistent_grid(laf_patches_kernel, LP_NT, 0, p.total), LP_NT, 0, st>>>(p);
  return launch_status("laf_patches_kernel");
}

}  // namespace kb200
