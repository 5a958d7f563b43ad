// kornia_b200 -- square 2-D correlation for odd K from 9 to 31 that skips the zero taps (fp32, 'same' padding).
//
// The large kernels behind filter2d are mostly zeros: a nearest-rotated motion-blur line (filters/motion.py) has about K to
// 1.4 K nonzero taps out of K^2, a bilinear one about 3 K.  The generic kernel (filter_generic.cuh) pays K^2 gathers per
// output regardless.  This kernel has the skeleton of filter2d_tiled_kernel -- persistent CTAs walk strips of 128 x 32
// tiles, the input box is TMA-loaded and double buffered behind an mbarrier, 'reflect' / 'replicate' patch the box on
// edge tiles only -- with one wide box for every K: 16 texels of padding left and right (>= the largest halo, and the
// TMA start stays 16-byte aligned), (32 + K - 1) rows.
//
// Tap list: when a CTA starts a strip whose sample uses another kernel than the last one (sample b uses kernel b mod Bk),
// warp 0 compacts that kernel's K x K taps in shared memory with ballots: the nonzero taps in row-major order, each as
// (weight, box offset).  Each thread owns a 4 x 4 set of outputs (rows 4 rg .. 4 rg + 3, columns q, q + 32, q + 64,
// q + 96, so a warp's shared loads are 32 consecutive words) and runs acc = fma(w, v, acc) over the list in order.
//
// Exactness: that is the generic kernel's sum with the terms fma(0, v, acc) left out, and leaving one out changes nothing
// unless v is non-finite (0 * Inf and 0 * NaN are NaN) or acc is -0 (-0 + +0 = +0).  acc starts at +0 and becomes -0
// only when an FMA rounds a nonzero exact result to zero.  If every product of a nonzero tap and a nonzero texel has
// magnitude >= 2^-100, every exact result is a multiple of 2^-149 (the products' granularity is at least
// |w| |v| 2^-48 >= 2^-148) and none rounds to zero.  So a tile whose box holds a non-finite texel, or a nonzero texel
// below 2^-100 / (the kernel's smallest nonzero |w|), runs the dense K^2 loop from the same box, in the generic kernel's
// order.  Either way the result is bit-identical to filter2d_fwd_generic for every input.  The guard scans the whole box,
// including cells no output reads; that can only send a tile to the dense loop, never away from it.
#pragma once
#include "sepfilter_tiled.cuh"

namespace kb200 {

constexpr int F2DT_KMIN = 9, F2DT_KMAX = 31;
constexpr int F2DT_XPAD = 16;                      // box columns left and right of the tile: >= the largest halo (15)
constexpr int F2DT_BW = SEPT_TW + 2 * F2DT_XPAD;  // 160
constexpr float F2DT_TINY = 0x1p-100f;             // the bound on |w| |v| of the exactness argument

struct F2dTapsParams {
  const float* k;  // (Bk, K, K)
  float* out;
  int C, H, W, Bk, planes, K;
};

// dynamic shared memory of one CTA: two boxes, two mbarriers, the tap list, the dense taps, the list length and bound
__host__ __device__ inline size_t f2d_taps_smem_bytes(int K) {
  return (size_t)2 * (SEPT_TH + K - 1) * F2DT_BW * 4 + 2 * sizeof(uint64_t) + (size_t)K * K * (sizeof(float2) + sizeof(float)) + 8;
}

// Warp 0: the nonzero taps of kernel `k` in row-major order as (w, offset of the tap in the box), every tap for the
// dense loop, the list length and the texel bound F2DT_TINY / min |w| (0 when the kernel has no nonzero tap).
__device__ __forceinline__ void f2d_compact_taps(const float* k, int K, float2* list, float* dense_k, int* n_taps, float* v_tiny) {
  const int lane = threadIdx.x & 31, KK = K * K;
  int n = 0;
  float wmin = INFINITY;
  for (int t0 = 0; t0 < KK; t0 += 32) {
    const int t = t0 + lane;
    const float w = t < KK ? __ldg(k + t) : 0.f;
    if (t < KK) dense_k[t] = w;
    const bool nz = w != 0.f;  // NaN counts as nonzero: it is kept, as the generic kernel's sum keeps it
    const unsigned m = __ballot_sync(0xffffffffu, nz);
    if (nz) {
      const int i = t / K;
      list[n + __popc(m & ((1u << lane) - 1u))] = make_float2(w, __int_as_float(i * F2DT_BW + (t - i * K)));
      wmin = fminf(wmin, fabsf(w));
    }
    n += __popc(m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmin = fminf(wmin, __shfl_xor_sync(0xffffffffu, wmin, o));
  if (lane == 0) {
    *n_taps = n;
    *v_tiny = F2DT_TINY / wmin;
  }
}

// A texel that could make skipping a zero tap observable (see the exactness note above).
__device__ __forceinline__ bool f2d_texel_unsafe(float v, float tiny) {
  const float a = fabsf(v);
  return !(a <= 3.40282347e38f) || (a != 0.f && a < tiny);
}

template <int BORDER>
__global__ void __launch_bounds__(256, 2) filter2d_taps_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ F2dTapsParams p) {
  constexpr int TW = SEPT_TW, TH = SEPT_TH, BW = F2DT_BW;
  static_assert(TW / 32 == 4 && TH / 4 == 8, "thread mapping: 32 lanes x 4 columns, 8 row groups x 4 rows");
  const int K = p.K, KK = K * K, HALO = (K - 1) / 2;
  const int BH = TH + K - 1;
  const int TILE_FLOATS = BH * BW;
  const uint32_t TILE_BYTES = (uint32_t)TILE_FLOATS * 4;

  extern __shared__ __align__(128) unsigned char f2dt_smem[];
  float* tiles = reinterpret_cast<float*>(f2dt_smem);  // [2][BH][BW]
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + 2 * TILE_FLOATS);
  float2* list = reinterpret_cast<float2*>(full + 2);  // [KK], the first *n_taps used
  float* dense_k = reinterpret_cast<float*>(list + KK);  // [KK]
  int* n_taps = reinterpret_cast<int*>(dense_k + KK);
  float* v_tiny = reinterpret_cast<float*>(n_taps + 1);

  const int tid = threadIdx.x;
  feed_init(full);

  const int tiles_x = ceil_div(p.W, TW), tiles_y = ceil_div(p.H, TH);
  const Segments segs(p.planes * tiles_y, tiles_x);

  TileFeed<false> feed(segs);
  auto load = [&](int slot, int strip, int tx, bool) {
    const int plane = strip / tiles_y, ty = strip - plane * tiles_y;
    tma::mbar_arrive_expect_tx(&full[slot], TILE_BYTES);
    tma::load_3d(tiles + slot * TILE_FLOATS, &tmap, &full[slot], tx * TW - F2DT_XPAD, ty * TH - HALO, plane);
  };
  if (tid == 0) feed.start(load);

  const int q = tid & 31, rg = tid >> 5;  // columns q + 32 c, rows 4 rg + o of the tile
  const int col0 = F2DT_XPAD - HALO;      // box column of the first tap of output column 0

  int cur_k = -1;
  int n = 0, strip, tx0, tx1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, tx0, tx1, cursor); ++seg) {
    const int plane = strip / tiles_y, ty = strip - plane * tiles_y;
    const int kb = (plane / p.C) % p.Bk;
    const int y0 = ty * TH;
    if (kb != cur_k) {  // CTA-uniform; every thread has passed the barrier after its last read of the old list
      if (tid < 32) f2d_compact_taps(p.k + (size_t)kb * KK, K, list, dense_k, n_taps, v_tiny);
      __syncthreads();
      cur_k = kb;
    }
    const int ntap = *n_taps;
    const float tiny = *v_tiny;
    float* orow = p.out + (size_t)plane * p.H * p.W + (size_t)(y0 + 4 * rg) * p.W + (size_t)tx0 * TW + q;
    const bool rows_full = y0 + TH <= p.H;

    for (int tx = tx0; tx < tx1; ++tx, ++n, orow += TW) {
      const int s = n & 1;
      float* tile = tiles + s * TILE_FLOATS;
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      patch_box_border<BORDER>(tile, BH, BW, tx * TW - F2DT_XPAD, y0 - HALO, p);

      bool unsafe = false;
      {
        const float4* t4 = reinterpret_cast<const float4*>(tile);
        for (int e = tid; e < TILE_FLOATS / 4; e += 256) {
          const float4 v = t4[e];
          unsafe |= f2d_texel_unsafe(v.x, tiny) | f2d_texel_unsafe(v.y, tiny) | f2d_texel_unsafe(v.z, tiny) | f2d_texel_unsafe(v.w, tiny);
        }
      }
      const bool dense = __syncthreads_or(unsafe) != 0;

      float acc[4][4];
#pragma unroll
      for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[o][c] = 0.f;
      const float* base = tile + (4 * rg) * BW + col0 + q;
      if (!dense) {
#pragma unroll 2
        for (int t = 0; t < ntap; ++t) {
          const float2 e = list[t];
          const float* src = base + __float_as_int(e.y);
#pragma unroll
          for (int o = 0; o < 4; ++o)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[o][c] = __fmaf_rn(e.x, src[o * BW + 32 * c], acc[o][c]);
        }
      } else {
        for (int i = 0; i < K; ++i)
          for (int j = 0; j < K; ++j) {
            const float w = dense_k[i * K + j];
            const float* src = base + i * BW + j;
#pragma unroll
            for (int o = 0; o < 4; ++o)
#pragma unroll
              for (int c = 0; c < 4; ++c) acc[o][c] = __fmaf_rn(w, src[o * BW + 32 * c], acc[o][c]);
          }
      }
      __syncthreads();  // tile[s] consumed by every thread
      if (tid == 0) feed.issue(load);

      if (rows_full && (tx + 1) * TW <= p.W) {
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
          for (int c = 0; c < 4; ++c) __stcs(orow + (size_t)o * p.W + 32 * c, acc[o][c]);
      } else {
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          if (y0 + 4 * rg + o >= p.H) continue;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (tx * TW + q + 32 * c < p.W) __stcs(orow + (size_t)o * p.W + 32 * c, acc[o][c]);
        }
      }
    }
  }
}

// KB200_EUNSUPPORTED unless K is odd in [9, 31], kh == kw, 'same' padding, a non-circular border, W % 4 == 0,
// 16-byte aligned x and out, and H, W > halo for 'reflect' / 'replicate'; the caller then runs filter2d_fwd_generic.
int filter2d_taps_forward(const float* x, const float* k, float* out, int B, int C, int H, int W, int Bk, int kh, int kw, int border,
                          int same, cudaStream_t st);

}  // namespace kb200
