// kornia_b200 -- host dispatch of the tiled small-kernel filter2d.
#include "filter2d_tiled.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

template <int K, int BORDER, bool DOWN2 = false>
static int launch_f2d_tiled(const CUtensorMap& map, const F2dTiledParams& p, cudaStream_t st) {
  constexpr size_t smem = f2d_tiled_smem_bytes<K>();
  auto kern = filter2d_tiled_kernel<K, BORDER, DOWN2>;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, smem);
  kern<<<capped_grid((long long)p.planes * ceil_div(p.H, SEPT_TH), 3), 256, smem, st>>>(map, p);
  return launch_status("filter2d_tiled");
}

// pyrdown in one pass (filter2d_tiled_kernel<5, BORDER, DOWN2 = true>).  KB200_EUNSUPPORTED -> the host composes
// filter2d + F.interpolate.
int pyrdown_tiled_forward(const float* x, const float* k, float* out, int B, int C, int H, int W, int Bk, int border, cudaStream_t st) {
  if (border == KB200_CIRCULAR || (H % 2) != 0 || (W % 4) != 0) return KB200_EUNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0) return KB200_EUNSUPPORTED;
  if (border != KB200_CONSTANT && (H <= 2 || W <= 2)) return KB200_EUNSUPPORTED;
  if ((long long)B * C * ceil_div(H, SEPT_TH) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  if (!encode_plane_map(&map, x, (long long)B * C, H, W, SEPT_BW, SEPT_TH + 4)) return KB200_EUNSUPPORTED;
  F2dTiledParams p{k, out, C, H, W, Bk, B * C};
  if (border == KB200_CONSTANT) return launch_f2d_tiled<5, KB200_CONSTANT, true>(map, p, st);
  if (border == KB200_REFLECT) return launch_f2d_tiled<5, KB200_REFLECT, true>(map, p, st);
  return launch_f2d_tiled<5, KB200_REPLICATE, true>(map, p, st);
}

// KB200_EUNSUPPORTED -> the caller runs filter2d_fwd_generic.
int filter2d_tiled_forward(const float* x, const float* k, float* out, int B, int C, int H, int W, int Bk, int kh, int kw, int border,
                           int same, cudaStream_t st) {
  if (!option(OPT_TILED_FILTER)) return KB200_EUNSUPPORTED;
  if (!same || kw != kh || (kw != 3 && kw != 5 && kw != 7) || border == KB200_CIRCULAR) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) return KB200_EUNSUPPORTED;
  const int halo = (kw - 1) / 2;
  if (border != KB200_CONSTANT && (H <= halo || W <= halo)) return KB200_EUNSUPPORTED;
  if ((long long)B * C * ceil_div(H, SEPT_TH) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  if (!encode_plane_map(&map, x, (long long)B * C, H, W, SEPT_BW, SEPT_TH + kw - 1)) return KB200_EUNSUPPORTED;
  F2dTiledParams p{k, out, C, H, W, Bk, B * C};
#define KB_F2D_CASE(K_)                                                                    \
  if (kw == K_) {                                                                          \
    if (border == KB200_CONSTANT) return launch_f2d_tiled<K_, KB200_CONSTANT>(map, p, st); \
    if (border == KB200_REFLECT) return launch_f2d_tiled<K_, KB200_REFLECT>(map, p, st);   \
    return launch_f2d_tiled<K_, KB200_REPLICATE>(map, p, st);                              \
  }
  KB_F2D_CASE(3)
  KB_F2D_CASE(5)
  KB_F2D_CASE(7)
#undef KB_F2D_CASE
  return KB200_EUNSUPPORTED;
}

}  // namespace kb200
