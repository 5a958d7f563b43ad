// kornia_b200 -- the TMA-tiled warp forward kernel with 32 x 32 output tiles and a 56 x 56 source box (bilinear,
// C in {1,3}).  The default 64 x 32 tile / 72 x 40 box serves near-identity maps (the headline homographies); a
// rotation by more than a few degrees turns the tile's footprint into a tall box that does not fit, and every pixel
// of the tile falls to the exact per-pixel path (measured: rotate by +-30 degrees ran at 20 % of the HBM roofline).
// A 32 x 32 tile rotated by any angle at unit scale covers at most 45 x 45 source pixels.  warp_tma.cu issues both
// kernels; each takes the samples of its footprint class (warp_tma.cuh: footprint_class) and skips the others.
#include "warp_tma_host.cuh"

namespace kb200 {

constexpr int SQ_TW = 32, SQ_TH = 32, SQ_BW = 56, SQ_BH = 56, SQ_STAGES = 2, SQ_CTAS = 2;

template <int NC, int PAD>
static int launch_square(const TmaBoxMaps& map, const TmaWarpParams& p, bool projective, bool align, cudaStream_t st) {
  if (projective)
    return align ? launch_warp_tma<NC, KB200_BILINEAR, PAD, true, true, SQ_TW, SQ_TH, SQ_BW, SQ_BH, SQ_STAGES>(map, p, st, SQ_CTAS)
                 : launch_warp_tma<NC, KB200_BILINEAR, PAD, true, false, SQ_TW, SQ_TH, SQ_BW, SQ_BH, SQ_STAGES>(map, p, st, SQ_CTAS);
  return align ? launch_warp_tma<NC, KB200_BILINEAR, PAD, false, true, SQ_TW, SQ_TH, SQ_BW, SQ_BH, SQ_STAGES>(map, p, st, SQ_CTAS)
               : launch_warp_tma<NC, KB200_BILINEAR, PAD, false, false, SQ_TW, SQ_TH, SQ_BW, SQ_BH, SQ_STAGES>(map, p, st, SQ_CTAS);
}

int warp_tma_forward_square(const TmaFwdArgs& a, cudaStream_t st) {
  if (a.C != 1 && a.C != 3) return KB200_EUNSUPPORTED;
  TmaBoxMaps map;
  if (!encode_box_maps<SQ_BW, SQ_BH>(map, a)) return KB200_EUNSUPPORTED;
  const TmaWarpParams p{a.src, a.m, a.bx, a.by, a.fill, a.out, a.B, a.H, a.W, a.h, a.w, a.Bm, a.align, a.only_class, nullptr};
  const bool projective = a.projective != 0, align = a.align != 0;
#define KB_SQ_CASE(NC_, PAD_) \
  if (a.C == NC_ && a.pad == PAD_) return launch_square<NC_, PAD_>(map, p, projective, align, st);
  KB_SQ_CASE(3, KB200_ZEROS)
  KB_SQ_CASE(3, KB200_BORDER)
  KB_SQ_CASE(3, KB200_REFLECTION)
  KB_SQ_CASE(3, KB200_FILL)
  KB_SQ_CASE(1, KB200_ZEROS)
  KB_SQ_CASE(1, KB200_BORDER)
  KB_SQ_CASE(1, KB200_REFLECTION)
  KB_SQ_CASE(1, KB200_FILL)
#undef KB_SQ_CASE
  return KB200_EUNSUPPORTED;
}

}  // namespace kb200
