// kornia_b200 -- host dispatch of the zero-skipping filter2d kernel (odd K from 9 to 31).
#include "filter2d_taps.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

template <int BORDER>
static int launch_f2d_taps(const CUtensorMap& map, const F2dTapsParams& p, cudaStream_t st) {
  auto kern = filter2d_taps_kernel<BORDER>;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, f2d_taps_smem_bytes(F2DT_KMAX));
  const size_t smem = f2d_taps_smem_bytes(p.K);
  // resident CTAs per SM for each K (shared memory decides: 4 at K = 9, 2 at K = 31)
  static int per_sm[F2DT_KMAX + 1] = {0};
  int ctas = __atomic_load_n(&per_sm[p.K], __ATOMIC_RELAXED);
  if (ctas == 0) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kern, 256, smem) != cudaSuccess || ctas < 1) ctas = 1;
    __atomic_store_n(&per_sm[p.K], ctas, __ATOMIC_RELAXED);
  }
  kern<<<capped_grid((long long)p.planes * ceil_div(p.H, SEPT_TH), ctas), 256, smem, st>>>(map, p);
  return launch_status("filter2d_taps");
}

int filter2d_taps_forward(const float* x, const float* k, float* out, int B, int C, int H, int W, int Bk, int kh, int kw, int border,
                          int same, cudaStream_t st) {
  if (!option(OPT_TILED_FILTER)) return KB200_EUNSUPPORTED;
  if (!same || kw != kh || (kw % 2) == 0 || kw < F2DT_KMIN || kw > F2DT_KMAX || border == KB200_CIRCULAR) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) return KB200_EUNSUPPORTED;
  const int halo = (kw - 1) / 2;
  if (border != KB200_CONSTANT && (H <= halo || W <= halo)) return KB200_EUNSUPPORTED;
  if ((long long)B * C * ceil_div(H, SEPT_TH) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  if (!encode_plane_map(&map, x, (long long)B * C, H, W, F2DT_BW, SEPT_TH + kw - 1)) return KB200_EUNSUPPORTED;
  F2dTapsParams p{k, out, C, H, W, Bk, B * C, kw};
  if (border == KB200_CONSTANT) return launch_f2d_taps<KB200_CONSTANT>(map, p, st);
  if (border == KB200_REFLECT) return launch_f2d_taps<KB200_REFLECT>(map, p, st);
  return launch_f2d_taps<KB200_REPLICATE>(map, p, st);
}

}  // namespace kb200
