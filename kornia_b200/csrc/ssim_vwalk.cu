// kornia_b200 -- host side of the band-walking SSIM kernel (ssim_vwalk.cuh).
#include "persistent_launch.cuh"
#include "ssim_vwalk.cuh"

namespace kb200 {

template <int K>
static int launch_ssimv(const CUtensorMap maps[4], const SsimVParams& p, cudaStream_t st) {
  auto kern = ssim_vwalk_kernel<K>;
  static unsigned long long configured = 0;
  KB_SET_SMEM_ONCE(configured, kern, ssimv_smem_bytes<K>());
  kern<<<capped_grid((long long)p.planes * ceil_div(p.W, VWALK_TW), 2), 256, ssimv_smem_bytes<K>(), st>>>(maps[0], maps[1], maps[2], maps[3], p);
  return launch_status("ssim_vwalk");
}

int ssim_vwalk_forward(const float* a, const float* b, const float* taps, float* out, int planes, int H, int W, int K, float C1, float C2,
                       float eps, cudaStream_t st) {
  if (K % 2 == 0 || K < 3 || K > SSIM_MAX_K || K / 2 >= H || K / 2 >= W) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(a) & 15) != 0 || (reinterpret_cast<uintptr_t>(b) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(out) & 7) != 0)
    return KB200_EUNSUPPORTED;
  if ((long long)planes * ceil_div(W, VWALK_TW) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  CUtensorMap maps[4];  // main a, main b, prologue a, prologue b
  for (int i = 0; i < 4; ++i)
    if (!encode_plane_map(&maps[i], (i & 1) ? b : a, planes, H, W, VWALK_BW, i < 2 ? VWALK_TH : K - 1)) return KB200_EUNSUPPORTED;
  SsimVParams p{taps, out, planes, H, W, C1, C2, eps};
  switch (K) {
    case 3: return launch_ssimv<3>(maps, p, st);
    case 5: return launch_ssimv<5>(maps, p, st);
    case 7: return launch_ssimv<7>(maps, p, st);
    case 9: return launch_ssimv<9>(maps, p, st);
    default: return launch_ssimv<11>(maps, p, st);
  }
}

}  // namespace kb200
