// kornia_b200 -- host side of the SIFT descriptor kernel (siftdesc.cuh).
#include "persistent_launch.cuh"
#include "siftdesc.cuh"

namespace kb200 {

int sift_describe_forward(const float* x, const float* gk, const float* pk, float* out, long long N, int P, long long sB, long long sH, int A,
                          int S, int K, int stride, int pad, int rootsift, float clipval, float eps, cudaStream_t st) {
  if (P > PH_MAX_P || K > PH_MAX_P || A * S * S > SIFT_MAX_D) return KB200_EUNSUPPORTED;
  SiftParams p{};
  p.src = x;
  p.gk = gk;
  p.pk = pk;
  p.out = out;
  p.sB = sB;
  p.sH = sH;
  p.N = N;
  p.P = P;
  p.A = A;
  p.S = S;
  p.K = K;
  p.stride = stride;
  p.pad = pad;
  p.rootsift = rootsift;
  p.clipval = clipval;
  p.eps = eps;
  const int smem = (int)sizeof(float) * sift_smem_floats(P, K, A * S * S);
  KB_CUDA(cudaFuncSetAttribute(sift_describe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  sift_describe_kernel<<<persistent_grid(sift_describe_kernel, PH_NT, smem, N), PH_NT, smem, st>>>(p);
  return launch_status("sift_describe_kernel");
}

}  // namespace kb200
