// kornia_b200 -- host helpers shared by the persistent-CTA launchers (nms.cu, quad_interp.cu).
#pragma once
#include "common.cuh"
#include "warp_tma.cuh"

namespace kb200 {

// Persistent grid: as many CTAs as fit on the device at once, or one per tile when there are fewer tiles.
template <typename Kern>
inline int persistent_grid(Kern kern, int threads, int smem, long long tiles) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const long long cap = (long long)per_sm * sm_count();
  return (int)(tiles < cap ? tiles : cap);
}

inline int launch_status(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s launch failed: %s", what, cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

}  // namespace kb200
