// kornia_b200 -- host dispatch of the tiled separable filter.
#include "persistent_launch.cuh"
#include "sepfilter_tiled.cuh"

namespace kb200 {

template <int K, int BORDER, bool LERP = false>
static int launch_sep_tiled(const CUtensorMap& map, const SepTiledParams& p, cudaStream_t st) {
  constexpr size_t smem = sept_smem_bytes<K>();
  auto kern = sepfilter_tiled_kernel<K, BORDER, LERP>;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, smem);
  kern<<<capped_grid((long long)p.planes * ceil_div(p.H, SEPT_TH), 3), 256, smem, st>>>(map, p);
  return launch_status("sepfilter_tiled");
}

// KB200_EUNSUPPORTED -> caller uses sepfilter_fwd_generic (circular border, 'valid', even / non-square /
// > 17-tap kernels, rows not 16-byte aligned, images narrower than the fold distance).
int sepfilter_tiled_forward(const float* x, const float* kx, const float* ky, float* out, int B, int C, int H, int W,
                                   int Bkx, int kw, int Bky, int kh, int border, int same, cudaStream_t st, const float* lerp_w) {
  if (!option(OPT_TILED_FILTER)) return KB200_EUNSUPPORTED;
  if (!same || kw != kh || (kw & 1) == 0 || kw < 3 || kw > 17 || border == KB200_CIRCULAR) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0) return KB200_EUNSUPPORTED;
  const int halo = (kw - 1) / 2;
  if (border != KB200_CONSTANT && (H <= halo || W <= halo)) return KB200_EUNSUPPORTED;  // fold source must be in the box
  if ((long long)B * C * ceil_div(H, SEPT_TH) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  if (!encode_plane_map(&map, x, (long long)B * C, H, W, SEPT_BW, SEPT_TH + kw - 1)) return KB200_EUNSUPPORTED;
  SepTiledParams p{kx, ky, out, C, H, W, Bkx, Bky, B * C, x, lerp_w ? *lerp_w : 0.f};
  if (lerp_w) {
    if (kw > 11 || (reinterpret_cast<uintptr_t>(x) & 7) != 0) return KB200_EUNSUPPORTED;
#define KB_SEP_LERP_CASE(K_)                                                                     \
  if (kw == K_) {                                                                                \
    if (border == KB200_CONSTANT) return launch_sep_tiled<K_, KB200_CONSTANT, true>(map, p, st); \
    if (border == KB200_REFLECT) return launch_sep_tiled<K_, KB200_REFLECT, true>(map, p, st);   \
    return launch_sep_tiled<K_, KB200_REPLICATE, true>(map, p, st);                              \
  }
    KB_SEP_LERP_CASE(3)
    KB_SEP_LERP_CASE(5)
    KB_SEP_LERP_CASE(7)
    KB_SEP_LERP_CASE(9)
    KB_SEP_LERP_CASE(11)
#undef KB_SEP_LERP_CASE
    return KB200_EUNSUPPORTED;
  }
#define KB_SEP_CASE(K_)                                                                    \
  if (kw == K_) {                                                                          \
    if (border == KB200_CONSTANT) return launch_sep_tiled<K_, KB200_CONSTANT>(map, p, st); \
    if (border == KB200_REFLECT) return launch_sep_tiled<K_, KB200_REFLECT>(map, p, st);   \
    return launch_sep_tiled<K_, KB200_REPLICATE>(map, p, st);                              \
  }
  KB_SEP_CASE(3)
  KB_SEP_CASE(5)
  KB_SEP_CASE(7)
  KB_SEP_CASE(9)
  KB_SEP_CASE(11)
  KB_SEP_CASE(13)
  KB_SEP_CASE(15)
  KB_SEP_CASE(17)
#undef KB_SEP_CASE
  return KB200_EUNSUPPORTED;
}

}  // namespace kb200
