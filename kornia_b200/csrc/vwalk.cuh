// kornia_b200 -- the band walk shared by ssim_vwalk_kernel and corner_vwalk_kernel: persistent CTAs of 256 threads walk
// 64-column bands top to bottom in 32-row tiles, row-filter each tile's boxes into Q planes of row sums and column-filter
// those with the K-tap window.  Shared memory holds the planes as mid[Q][MH][VWALK_TW], MH = VWALK_TH + K - 1 rows: mid row
// 0 is image row t * VWALK_TH - K / 2 of tile t.  The K - 1 rows shared by vertically adjacent tiles stay in mid from one
// tile to the next, so every row is row-filtered once.  Each kernel keeps its own row pass and its own epilogue.
#pragma once
#include "tile_feed.cuh"

namespace kb200 {

constexpr int VWALK_TW = 64;                          // band width
constexpr int VWALK_TH = 32;                          // tile rows
constexpr int VWALK_XPAD = 8;                         // box columns left and right of the band
constexpr int VWALK_BW = VWALK_TW + 2 * VWALK_XPAD;   // 80
constexpr int VWALK_QUADS = VWALK_TW / 4;             // row pass: 16 quads per row
constexpr int VWALK_RPS = 256 / VWALK_QUADS;          // 16 rows per sweep of the CTA
constexpr int VWALK_SWEEPS = VWALK_TH / VWALK_RPS;    // 2
constexpr int VWALK_RY = 4;                           // column pass: rows per thread
static_assert((VWALK_TW / 2) * (VWALK_TH / VWALK_RY) == 256 && VWALK_SWEEPS * VWALK_RPS == VWALK_TH, "thread mapping");

// First / last tiles of a band (CTA-uniform test): mid rows outside the image (gy0 is the image row of mid row 0) become
// copies of their reflections, then the CTA synchronises.  The reflected row is an in-image row, which this never writes.
template <int Q, int K>
__device__ __forceinline__ void vwalk_reflect_rows(float4* mid4, int gy0, int H) {
  constexpr int MH = VWALK_TH + K - 1, QUADS = VWALK_QUADS;
  if (gy0 < 0 || gy0 + MH > H) {
    for (int e = threadIdx.x; e < MH * QUADS; e += 256) {
      const int mr = e / QUADS, qd = e - mr * QUADS;
      const int gy = gy0 + mr;
      if ((unsigned)gy < (unsigned)H) continue;
      const int sr = border_index<KB200_REFLECT>(gy, H) - gy0;
      if ((unsigned)sr < (unsigned)MH) {
#pragma unroll
        for (int q = 0; q < Q; ++q) mid4[(q * MH + mr) * QUADS + qd] = mid4[(q * MH + sr) * QUADS + qd];
      }
    }
    __syncthreads();
  }
}

// Column pass of thread (cp, rg): column pair cp, tile rows rg * RY .. + RY - 1 of every plane, ascending taps, two FFMAs
// per pair (fma2_rn).
template <int Q, int K>
__device__ __forceinline__ void vwalk_column_pass(const float* mid, const float (&k)[K], int cp, int rg, float2 (&acc)[Q][VWALK_RY]) {
  constexpr int MH = VWALK_TH + K - 1, TW = VWALK_TW, RY = VWALK_RY;
#pragma unroll
  for (int q = 0; q < Q; ++q)
#pragma unroll
    for (int o = 0; o < RY; ++o) acc[q][o] = make_float2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < RY + K - 1; ++i) {
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const float2 v = *reinterpret_cast<const float2*>(mid + (q * MH + rg * RY + i) * TW + 2 * cp);
#pragma unroll
      for (int o = 0; o < RY; ++o) {
        if (i - o >= 0 && i - o < K) acc[q][o] = fma2_rn(make_float2(k[i - o], k[i - o]), v, acc[q][o]);
      }
    }
  }
}

// Carry rows [TH, MH) -> [0, K - 1) of the Q planes for the next tile: thread (rq, rr) of the row pass moves exactly the
// cells it overwrites in the next row pass (mid row K - 1 + rr + 16 * it, quad rq).
template <int Q, int K>
__device__ __forceinline__ void vwalk_carry_rows(float4* mid4, int rq, int rr) {
  constexpr int MH = VWALK_TH + K - 1, CARRY = K - 1, TH = VWALK_TH, QUADS = VWALK_QUADS;
  static_assert(CARRY <= VWALK_RPS, "one sweep carries every row");
#pragma unroll
  for (int it = 0; it < VWALK_SWEEPS; ++it) {
    const int R = CARRY + rr + it * VWALK_RPS;
    if (R >= TH) {
#pragma unroll
      for (int q = 0; q < Q; ++q) mid4[(q * MH + R - TH) * QUADS + rq] = mid4[(q * MH + R) * QUADS + rq];
    }
  }
}

}  // namespace kb200
