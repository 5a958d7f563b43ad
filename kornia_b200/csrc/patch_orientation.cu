// kornia_b200 -- host side of the dominant-orientation kernel (patch_orientation.cuh).
#include "patch_orientation.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

int patch_orientation_forward(const float* x, const float* weighting, const float* smooth, float* out, long long N, int P, long long sB,
                              long long sH, int A, float eps, cudaStream_t st) {
  if (P > PH_MAX_P || A < 2 || A > ORI_MAX_BINS) return KB200_EUNSUPPORTED;
  OriParams p{};
  p.src = x;
  p.weighting = weighting;
  p.smooth = smooth;
  p.out = out;
  p.sB = sB;
  p.sH = sH;
  p.N = N;
  p.P = P;
  p.A = A;
  p.eps = eps;
  const int smem = (int)sizeof(float) * ori_smem_floats(P, A);
  KB_CUDA(cudaFuncSetAttribute(patch_orientation_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  patch_orientation_kernel<<<persistent_grid(patch_orientation_kernel, PH_NT, smem, N), PH_NT, smem, st>>>(p);
  return launch_status("patch_orientation_kernel");
}

}  // namespace kb200
