// kornia_b200 -- host side of the band-walking Harris / GFTT kernel (corner_vwalk.cuh).
#include "corner_vwalk.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

template <int KIND>
static int launch_corner(const CUtensorMap maps[2], const CornerParams& p, cudaStream_t st) {
  auto kern = corner_vwalk_kernel<KIND>;
  static unsigned long long configured = 0;
  KB_SET_SMEM_ONCE(configured, kern, corner_smem_bytes());
  kern<<<capped_grid((long long)p.planes * ceil_div(p.W, VWALK_TW), 2), 256, corner_smem_bytes(), st>>>(maps[0], maps[1], p);
  return launch_status("corner_vwalk");
}

int corner_vwalk_forward(const float* x, const double* stencil, const float* taps, float k, const float* kptr, const float* s4, float* out,
                         int planes, int C, int H, int W, int kind, cudaStream_t st) {
  if (kind != RESP_HARRIS && kind != RESP_GFTT) return KB200_EUNSUPPORTED;
  if (H <= CORNER_K / 2 || W <= CORNER_K / 2) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0) return KB200_EUNSUPPORTED;
  if ((long long)planes * ceil_div(W, VWALK_TW) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  CUtensorMap maps[2];  // main (TH + 2 rows), prologue (K - 1 + 2 rows)
  for (int i = 0; i < 2; ++i)
    if (!encode_plane_map(&maps[i], x, planes, H, W, VWALK_BW, i == 0 ? VWALK_TH + 2 : CORNER_K - 1 + 2)) return KB200_EUNSUPPORTED;
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
