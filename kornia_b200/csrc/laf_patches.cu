// kornia_b200 -- host side of the LAF patch extraction kernel (laf_patches.cuh).
#include "laf_patches.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

int extract_patches_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                            void* out, long long B, long long N, int C, int PS, int normalize, int select_level, cudaStream_t st) {
  KB_CHECK_ARG(n_levels >= 1 && n_levels <= LP_MAX_LEVELS && (select_level || n_levels == 1), "bad level count %d", n_levels);
  LafPatchParams p{};
  const int rc = laf_level_table(p, levels, level_dims, n_levels, PS, B * N > 0 && normalize);  // checked even with no patches
  if (rc != KB200_OK || B * N == 0) return rc;
  KB_CHECK_ARG(laf && base && out, "null pointer argument");
  p.laf = (const float*)laf;
  p.base = (const float*)base;
  p.out = (float*)out;
  p.N = N;
  p.total = B * N;
  p.C = C;
  p.PS = PS;
  p.normalize = normalize;
  p.select_level = select_level;
  laf_patches_kernel<<<persistent_grid(laf_patches_kernel, LP_NT, 0, p.total), LP_NT, 0, st>>>(p);
  return launch_status("laf_patches_kernel");
}

}  // namespace kb200
