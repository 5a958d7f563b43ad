// kornia_b200 -- small square 2-D correlation, one pass over HBM (fp32, 'same' padding, K in {3,5,7}).
//
// Replaces F.pad + grouped F.conv2d of kornia/filters/filter.py:136-150 for the kernels behind sobel /
// laplacian / box_blur / unsharp / gaussian_blur2d(separable=False).  Same skeleton as the separable
// kernel (sepfilter_tiled.cuh): persistent CTAs walk strips of 128 x 32 tiles, the (128+16) x (32+K-1)
// input box is TMA-loaded and double buffered, borders come from zero fill ('constant') or from a
// patch of the box on edge tiles ('reflect' / 'replicate').  Each thread produces a 4 x 4 block of
// outputs from a (4+K-1)-row register window (aligned LDS.128), K*K FMAs per output, taps in
// registers for the whole strip, tap order row-major ascending = the generic kernel's (bit-identical).
//
// DOWN2 (pyrdown, kornia/geometry/transform/pyramid.py:444-457): the epilogue averages each 2 x 2 block of the
// thread's 4 x 4 filtered outputs and writes the (H/2, W/2) image -- F.interpolate(bilinear, align_corners=False) at an
// exact factor of two samples at 2 d + 0.5, i.e. both lambdas are 1/2 and ATen's
// h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d) is 0.25 * ((a + b) + (c + d)) with one rounding per add (scaling by
// a power of two is exact, with or without FMA contraction).  The filtered full-size image never reaches HBM:
// 4 B read + 1 B written per input element instead of 8 + 5.
#pragma once
#include "sepfilter_tiled.cuh"

namespace kb200 {

struct F2dTiledParams {
  const float* k;  // (Bk, K, K)
  float* out;
  int C, H, W, Bk, planes;
};

template <int K>
constexpr size_t f2d_tiled_smem_bytes() {  // two boxes, two mbarriers
  return (size_t)(2 * (SEPT_TH + K - 1) * SEPT_BW) * 4 + 2 * sizeof(uint64_t);
}

template <int K, int BORDER, bool DOWN2 = false>
__global__ void __launch_bounds__(256, 3) filter2d_tiled_kernel(const __grid_constant__ CUtensorMap tmap,
                                                                const __grid_constant__ F2dTiledParams p) {
  constexpr int HALO = (K - 1) / 2;
  constexpr int TW = SEPT_TW, TH = SEPT_TH, BW = SEPT_BW;
  constexpr int BH = TH + K - 1;
  constexpr int COL0 = SEPT_XPAD - HALO;
  constexpr int A0 = COL0 & 3;
  constexpr int NV = (A0 + 4 + K - 1 + 3) / 4;
  constexpr int TILE_FLOATS = BH * BW;
  constexpr uint32_t TILE_BYTES = TILE_FLOATS * 4;
  static_assert(TW / 4 == 32 && TH / 4 == 8, "thread mapping: 32 quads x 8 row groups");

  extern __shared__ __align__(128) unsigned char f2d_smem[];  // f2d_tiled_smem_bytes<K>()
  float* tiles = reinterpret_cast<float*>(f2d_smem);  // [2][BH][BW]
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + 2 * TILE_FLOATS);

  const int tid = threadIdx.x;
  feed_init(full);

  const int tiles_x = ceil_div(p.W, TW), tiles_y = ceil_div(p.H, TH);
  const Segments segs(p.planes * tiles_y, tiles_x);

  TileFeed<false> feed(segs);
  auto load = [&](int slot, int strip, int tx, bool) {
    const int plane = strip / tiles_y, ty = strip - plane * tiles_y;
    tma::mbar_arrive_expect_tx(&full[slot], TILE_BYTES);
    tma::load_3d(tiles + slot * TILE_FLOATS, &tmap, &full[slot], tx * TW - SEPT_XPAD, ty * TH - HALO, plane);
  };
  if (tid == 0) feed.start(load);

  const int q = tid & 31, rg = tid >> 5;  // quad q (columns 4q..4q+3) of rows 4*rg .. 4*rg+3

  int n = 0, strip, tx0, tx1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, tx0, tx1, cursor); ++seg) {
    const int plane = strip / tiles_y, ty = strip - plane * tiles_y;
    const int b = plane / p.C;
    const int y0 = ty * TH;
    float kk[K * K];
#pragma unroll
    for (int i = 0; i < K * K; ++i) kk[i] = __ldg(p.k + (size_t)(b % p.Bk) * K * K + i);
    // DOWN2: the output plane is (H/2, W/2) (H even, W % 4 == 0: whole 2 x 2 blocks only) and a thread owns 2 x 2 of it
    float* orow = DOWN2 ? p.out + (size_t)plane * (p.H / 2) * (p.W / 2) + (size_t)(y0 / 2 + 2 * rg) * (p.W / 2) + (size_t)tx0 * (TW / 2) + 2 * q
                        : p.out + (size_t)plane * p.H * p.W + (size_t)(y0 + 4 * rg) * p.W + (size_t)tx0 * TW + 4 * q;
    const bool rows_full = y0 + TH <= p.H;

    for (int tx = tx0; tx < tx1; ++tx, ++n, orow += (DOWN2 ? TW / 2 : TW)) {
      const int s = n & 1;
      float* tile = tiles + s * TILE_FLOATS;
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      patch_box_border<BORDER>(tile, BH, BW, tx * TW - SEPT_XPAD, y0 - HALO, p);

      // 4 x 4 outputs per thread; rows enter the register window one at a time, each feeding up to K output rows
      float acc[4][4];
#pragma unroll
      for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int x = 0; x < 4; ++x) acc[o][x] = 0.f;
      const float4* src4 = reinterpret_cast<const float4*>(tile + (4 * rg) * BW + (COL0 & ~3) + 4 * q);
#pragma unroll
      for (int r = 0; r < 4 + K - 1; ++r) {
        float win[NV * 4];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const float4 t = src4[r * (BW / 4) + v];
          win[4 * v] = t.x; win[4 * v + 1] = t.y; win[4 * v + 2] = t.z; win[4 * v + 3] = t.w;
        }
        // window row r is tap row i = r - o of output row o.  For a fixed output the taps must accumulate in
        // row-major order (i ascending, then j): rows arrive in ascending r, so i ascends for every o.
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const int i = r - o;
          if (i >= 0 && i < K) {
#pragma unroll
            for (int j = 0; j < K; ++j)
#pragma unroll
              for (int x = 0; x < 4; ++x) acc[o][x] = __fmaf_rn(kk[i * K + j], win[A0 + x + j], acc[o][x]);
          }
        }
      }
      __syncthreads();  // tile[s] consumed by every thread
      if (tid == 0) feed.issue(load);

      if (DOWN2) {
        if (tx * TW + 4 * q < p.W) {
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            if (y0 + 4 * rg + 2 * o < p.H) {
              const float lo = 0.25f * __fadd_rn(__fadd_rn(acc[2 * o][0], acc[2 * o][1]), __fadd_rn(acc[2 * o + 1][0], acc[2 * o + 1][1]));
              const float hi = 0.25f * __fadd_rn(__fadd_rn(acc[2 * o][2], acc[2 * o][3]), __fadd_rn(acc[2 * o + 1][2], acc[2 * o + 1][3]));
              __stcs(reinterpret_cast<float2*>(orow + (size_t)o * (p.W / 2)), make_float2(lo, hi));
            }
          }
        }
      } else if (rows_full && (tx + 1) * TW <= p.W) {
        float* op = orow;
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          __stcs(reinterpret_cast<float4*>(op), make_float4(acc[o][0], acc[o][1], acc[o][2], acc[o][3]));
          op += p.W;
        }
      } else if (tx * TW + 4 * q < p.W) {
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          if (y0 + 4 * rg + o < p.H) __stcs(reinterpret_cast<float4*>(orow + (size_t)o * p.W), make_float4(acc[o][0], acc[o][1], acc[o][2], acc[o][3]));
        }
      }
    }
  }
}

int filter2d_tiled_forward(const float* x, const float* k, float* out, int B, int C, int H, int W, int Bk, int kh, int kw, int border,
                           int same, cudaStream_t st);
// 5 x 5 filter + 2 x 2 average in one pass: out (B,C,H/2,W/2).  KB200_EUNSUPPORTED unless H is even, W % 4 == 0 and the
// pointers are 16 / 8-byte aligned.
int pyrdown_tiled_forward(const float* x, const float* k, float* out, int B, int C, int H, int W, int Bk, int border, cudaStream_t st);

}  // namespace kb200
