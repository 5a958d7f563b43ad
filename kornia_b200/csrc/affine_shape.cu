// kornia_b200 -- host side of the affine shape kernels (affine_shape.cuh).
#include "affine_shape.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

int patch_affine_shape_forward(const float* x, const float* weighting, float* out, long long N, int P, long long sB, long long sH, float eps,
                               cudaStream_t st) {
  if (P > PH_MAX_P) return KB200_EUNSUPPORTED;
  PatchAffParams p{x, weighting, out, sB, sH, N, P, eps};
  const int smem = aff_smem_bytes(P);
  patch_affine_shape_kernel<<<persistent_grid(patch_affine_shape_kernel, PH_NT, smem, N), PH_NT, smem, st>>>(p);
  return launch_status("patch_affine_shape_kernel");
}

int laf_affine_shape_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                             const void* weighting, void* out, long long B, long long N, int PS, float eps, int preserve_orientation,
                             cudaStream_t st) {
  if (PS > PH_MAX_P) return KB200_EUNSUPPORTED;
  KB_CHECK_ARG(n_levels >= 1 && n_levels <= LP_MAX_LEVELS, "bad level count %d", n_levels);
  LafAffParams p{};
  const int rc = laf_level_table(p, levels, level_dims, n_levels, PS, B * N > 0);  // checked even with no keypoints
  if (rc != KB200_OK || B * N == 0) return rc;
  KB_CHECK_ARG(laf && base && weighting && out, "null pointer argument");
  p.laf = (const float*)laf;
  p.base = (const float*)base;
  p.weighting = (const float*)weighting;
  p.out = (float*)out;
  p.N = N;
  p.total = B * N;
  p.PS = PS;
  p.eps = eps;
  p.preserve_orientation = preserve_orientation;
  const int smem = aff_smem_bytes(PS);
  laf_affine_shape_kernel<<<persistent_grid(laf_affine_shape_kernel, PH_NT, smem, p.total), PH_NT, smem, st>>>(p);
  return launch_status("laf_affine_shape_kernel");
}

}  // namespace kb200
