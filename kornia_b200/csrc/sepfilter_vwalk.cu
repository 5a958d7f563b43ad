// kornia_b200 -- host dispatch of the band-walking separable filter (sepfilter_vwalk.cuh).
#include "sepfilter_vwalk.cuh"

namespace kb200 {

template <int K, int BORDER, bool LERP = false>
static int launch_sep_vwalk(const CUtensorMap& map_main, const CUtensorMap& map_pro, const SepTiledParams& p, cudaStream_t st) {
  constexpr size_t smem = (size_t)(2 * SEPT_TH * SEPT_BW + (SEPT_TH + K - 1) * SEPT_TW) * 4 + 2 * sizeof(uint64_t);
  auto kern = sepfilter_vwalk_kernel<K, BORDER, LERP>;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, smem);
  const long long nbands = (long long)p.planes * ceil_div(p.W, SEPT_TW);
  const long long cap = 3ll * sm_count();
  const int grid = (int)(nbands < cap ? nbands : cap);
  kern<<<grid, 256, smem, st>>>(map_main, map_pro, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sepfilter_vwalk launch failed: %s", cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

int sepfilter_vwalk_forward(const float* x, const float* kx, const float* ky, float* out, int B, int C, int H, int W, int Bkx, int kw,
                            int Bky, int kh, int border, int same, cudaStream_t st, const float* lerp_w) {
  // -1 = from 11 taps up, without the lerp epilogue of unsharp_mask.  Not the default: on an H100 SXM (700 W, B=256x3x1080x1920)
  // the tiled kernel was faster at 5-13 taps (k=11: 5.20 vs 5.66 ms) and equal at 17 (tools/ab_blur.py, both kernels interleaved).
  const int sel = option(OPT_SEP_VWALK);
  if (sel == 0 || (sel < 0 && (kw < 11 || lerp_w)) || !option(OPT_TILED_FILTER)) return KB200_EUNSUPPORTED;
  if (!same || kw != kh || (kw & 1) == 0 || kw < 3 || kw > 17 || border == KB200_CIRCULAR) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0) return KB200_EUNSUPPORTED;
  const int halo = (kw - 1) / 2;
  if (border != KB200_CONSTANT && (H <= halo || W <= halo)) return KB200_EUNSUPPORTED;  // fold sources must be real rows / columns
  if ((long long)B * C * ceil_div(W, SEPT_TW) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return KB200_EUNSUPPORTED;
  CUtensorMap map_main, map_pro;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B * C};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
  const cuuint32_t estr[3] = {1, 1, 1};
  const cuuint32_t box_main[3] = {(cuuint32_t)SEPT_BW, (cuuint32_t)SEPT_TH, 1};
  const cuuint32_t box_pro[3] = {(cuuint32_t)SEPT_BW, (cuuint32_t)(kw - 1), 1};
  if (encode(&map_main, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box_main, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return KB200_EUNSUPPORTED;
  if (encode(&map_pro, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box_pro, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return KB200_EUNSUPPORTED;
  SepTiledParams p{kx, ky, out, C, H, W, Bkx, Bky, B * C, x, lerp_w ? *lerp_w : 0.f};
  if (lerp_w) {  // unsharp_mask: the same envelope as the strip-walking lerp kernel
    if (kw > 11 || (reinterpret_cast<uintptr_t>(x) & 7) != 0) return KB200_EUNSUPPORTED;
#define KB_SEPV_LERP_CASE(K_)                                                                                  \
  if (kw == K_) {                                                                                              \
    if (border == KB200_CONSTANT) return launch_sep_vwalk<K_, KB200_CONSTANT, true>(map_main, map_pro, p, st); \
    if (border == KB200_REFLECT) return launch_sep_vwalk<K_, KB200_REFLECT, true>(map_main, map_pro, p, st);   \
    return launch_sep_vwalk<K_, KB200_REPLICATE, true>(map_main, map_pro, p, st);                              \
  }
    KB_SEPV_LERP_CASE(3)
    KB_SEPV_LERP_CASE(5)
    KB_SEPV_LERP_CASE(7)
    KB_SEPV_LERP_CASE(9)
    KB_SEPV_LERP_CASE(11)
#undef KB_SEPV_LERP_CASE
    return KB200_EUNSUPPORTED;
  }
#define KB_SEPV_CASE(K_)                                                                              \
  if (kw == K_) {                                                                                     \
    if (border == KB200_CONSTANT) return launch_sep_vwalk<K_, KB200_CONSTANT>(map_main, map_pro, p, st); \
    if (border == KB200_REFLECT) return launch_sep_vwalk<K_, KB200_REFLECT>(map_main, map_pro, p, st);   \
    return launch_sep_vwalk<K_, KB200_REPLICATE>(map_main, map_pro, p, st);                              \
  }
  KB_SEPV_CASE(3)
  KB_SEPV_CASE(5)
  KB_SEPV_CASE(7)
  KB_SEPV_CASE(9)
  KB_SEPV_CASE(11)
  KB_SEPV_CASE(13)
  KB_SEPV_CASE(15)
  KB_SEPV_CASE(17)
#undef KB_SEPV_CASE
  return KB200_EUNSUPPORTED;
}

}  // namespace kb200
