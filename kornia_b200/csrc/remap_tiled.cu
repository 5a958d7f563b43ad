// kornia_b200 -- host dispatch of the tiled remap forward kernel.
#include "persistent_launch.cuh"
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
  return launch_status("remap_tiled");
}

// KB200_EUNSUPPORTED -> the caller runs the generic kernel.
int remap_tiled_forward(const float* src, const float* map_x, const float* map_y, float* out, int B, int C, int H, int W, int h, int w,
                        int Bmap, int normalized, int interp, int pad, int align, cudaStream_t st) {
  if (!option(OPT_TMA)) return KB200_EUNSUPPORTED;
  if (interp != KB200_BILINEAR || (C != 1 && C != 3) || pad == KB200_FILL) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(src) & 15) != 0) return KB200_EUNSUPPORTED;
  if (B > 65535 || ceil_div(h, 32) > 65535) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  if (!encode_plane_map(&map, src, (long long)B * C, H, W, 72, 40, C)) return KB200_EUNSUPPORTED;
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
  CUtensorMap map;
  if (!encode_plane_map(&map, src, (long long)B * C, H, W, 72, 40, C)) return KB200_EUNSUPPORTED;
  RemapTiledParams p{src, nullptr, nullptr, out, B, H, W, H, W, B, 0, lens};
  return C == 3 ? launch_remap_tiled<3, KB200_ZEROS, true, true>(map, p, st) : launch_remap_tiled<1, KB200_ZEROS, true, true>(map, p, st);
}

}  // namespace kb200
