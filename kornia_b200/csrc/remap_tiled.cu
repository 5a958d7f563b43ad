// kornia_b200 -- host dispatch of the tiled remap forward kernel.
#include "remap_tiled.cuh"

namespace kb200 {

template <int NC, int PAD, bool ALIGN, bool LENS = false>
static int launch_remap_tiled(const CUtensorMap& map, const RemapTiledParams& p, cudaStream_t st) {
  auto kern = remap_tiled_kernel<NC, PAD, ALIGN, LENS>;
  constexpr size_t smem = (size_t)NC * 72 * 40 * 4 + 8 + 32 * 4 + 4 * 4 + 16;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, smem);
  const dim3 grid(ceil_div(p.w, 64), ceil_div(p.h, 32), p.B);
  kern<<<grid, 256, smem, st>>>(map, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("remap_tiled launch failed: %s", cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

// KB200_EUNSUPPORTED -> the caller runs the generic kernel.
int remap_tiled_forward(const float* src, const float* map_x, const float* map_y, float* out, int B, int C, int H, int W, int h, int w,
                        int Bmap, int normalized, int interp, int pad, int align, cudaStream_t st) {
  if (!option(OPT_TMA)) return KB200_EUNSUPPORTED;
  if (interp != KB200_BILINEAR || (C != 1 && C != 3) || pad == KB200_FILL) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(src) & 15) != 0) return KB200_EUNSUPPORTED;
  if (B > 65535 || ceil_div(h, 32) > 65535) return KB200_EUNSUPPORTED;
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B * C};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
  const cuuint32_t box[3] = {72, 40, (cuuint32_t)C};
  const cuuint32_t estr[3] = {1, 1, 1};
  if (encode(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(src), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return KB200_EUNSUPPORTED;
  RemapTiledParams p{src, map_x, map_y, out, B, H, W, h, w, Bmap, normalized, nullptr};
#define KB_REMAP_CASE(NC_, PAD_)                                                         \
  if (C == NC_ && pad == PAD_)                                                           \
    return align ? launch_remap_tiled<NC_, PAD_, true>(map, p, st) : launch_remap_tiled<NC_, PAD_, false>(map, p, st);
  KB_REMAP_CASE(3, KB200_ZEROS)
  KB_REMAP_CASE(3, KB200_BORDER)
  KB_REMAP_CASE(3, KB200_REFLECTION)
  KB_REMAP_CASE(1, KB200_ZEROS)
  KB_REMAP_CASE(1, KB200_BORDER)
  KB_REMAP_CASE(1, KB200_REFLECTION)
#undef KB_REMAP_CASE
  return KB200_EUNSUPPORTED;
}

// KB200_EUNSUPPORTED -> the host builds the maps with torch ops and calls kb200_remap_forward.
int undistort_tiled_forward(const float* src, const float* lens, float* out, int B, int C, int H, int W, cudaStream_t st) {
  if ((C != 1 && C != 3) || (W % 4) != 0 || (reinterpret_cast<uintptr_t>(src) & 15) != 0 || B > 65535 || ceil_div(H, 32) > 65535)
    return KB200_EUNSUPPORTED;
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B * C};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
  const cuuint32_t box[3] = {72, 40, (cuuint32_t)C};
  const cuuint32_t estr[3] = {1, 1, 1};
  if (encode(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(src), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return KB200_EUNSUPPORTED;
  RemapTiledParams p{src, nullptr, nullptr, out, B, H, W, H, W, B, 0, lens};
  return C == 3 ? launch_remap_tiled<3, KB200_ZEROS, true, true>(map, p, st) : launch_remap_tiled<1, KB200_ZEROS, true, true>(map, p, st);
}

}  // namespace kb200
