// kornia_b200 -- host helpers shared by the persistent-CTA launchers.
#pragma once
#include "common.cuh"
#include "tma.cuh"

namespace kb200 {

// ctas_per_sm CTAs on every SM, or one per unit of work when there is less work.
inline int capped_grid(long long work, int ctas_per_sm) {
  const long long cap = (long long)ctas_per_sm * sm_count();
  return (int)(work < cap ? work : cap);
}

// Persistent grid: as many CTAs as fit on the device at once, or one per tile when there are fewer tiles.
template <typename Kern>
inline int persistent_grid(Kern kern, int threads, int smem, long long tiles) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return capped_grid(tiles, per_sm);
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
