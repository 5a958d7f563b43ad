// kornia_b200 -- host side of the band-walking Harris / GFTT kernel (corner_vwalk.cuh).
#include "corner_vwalk.cuh"

namespace kb200 {

template <int KIND>
static int launch_corner(const CUtensorMap maps[2], const CornerParams& p, cudaStream_t st) {
  auto kern = corner_vwalk_kernel<KIND>;
  static unsigned long long configured = 0;
  KB_SET_SMEM_ONCE(configured, kern, corner_smem_bytes());
  const long long nbands = (long long)p.planes * ceil_div(p.W, SSIMV_TW);
  const long long cap = 2ll * sm_count();
  const int grid = (int)(nbands < cap ? nbands : cap);
  kern<<<grid, 256, corner_smem_bytes(), st>>>(maps[0], maps[1], p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("corner_vwalk launch failed: %s", cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

int corner_vwalk_forward(const float* x, const double* stencil, const float* taps, float k, const float* kptr, const float* s4, float* out,
                         int planes, int C, int H, int W, int kind, cudaStream_t st) {
  if (kind != RESP_HARRIS && kind != RESP_GFTT) return KB200_EUNSUPPORTED;
  if (H <= CORNER_K / 2 || W <= CORNER_K / 2) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0) return KB200_EUNSUPPORTED;
  if ((long long)planes * ceil_div(W, SSIMV_TW) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return KB200_EUNSUPPORTED;
  CUtensorMap maps[2];  // main (TH + 2 rows), prologue (K - 1 + 2 rows)
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
  const cuuint32_t estr[3] = {1, 1, 1};
  for (int i = 0; i < 2; ++i) {
    const cuuint32_t box[3] = {(cuuint32_t)SSIMV_BW, (cuuint32_t)(i == 0 ? SSIMV_TH + 2 : CORNER_K - 1 + 2), 1};
    if (encode(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return KB200_EUNSUPPORTED;
  }
  CornerParams p;
  p.taps = taps;
  p.kptr = kptr;
  p.s4 = s4;
  p.out = out;
  p.planes = planes;
  p.C = C;
  p.H = H;
  p.W = W;
  p.k = k;
  for (int e = 0; e < 2 * 9; ++e) p.st[e] = (float)stencil[e];  // exact: the host built them in fp32
  return kind == RESP_HARRIS ? launch_corner<RESP_HARRIS>(maps, p, st) : launch_corner<RESP_GFTT>(maps, p, st);
}

}  // namespace kb200
