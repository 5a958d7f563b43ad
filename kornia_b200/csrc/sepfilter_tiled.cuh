// kornia_b200 -- separable K x K filter, one pass over HBM (fp32, 'same' padding; the blur kernel).
//
// Replaces filter2d_separable's two (F.pad copy + grouped conv2d) passes (kornia/filters/filter.py:
// 205-207 -> :136-150) for square odd kernels: gaussian_blur2d(separable=True), SSIM windows, box blurs.
//
// Persistent CTAs (256 threads) walk strips of 128 x 32 output tiles of one plane, left to right:
//   1. TMA (cp.async.bulk.tensor) lands the (128+16) x (32+K-1) input box in shared memory, double
//      buffered: the box of tile t+1 is in flight while tile t is filtered.  Texels outside the image
//      arrive as zeros ('constant' border for free).  For 'reflect' / 'replicate' only tiles that touch
//      the image border patch their out-of-image halo cells from cells of the same box.
//   2. row pass: thread (q, r0) slides a K-tap window over 4 consecutive outputs of rows r0, r0+8, ...
//      (aligned LDS.128 in, 4 x K FMAs, STS.128 out; all shared addresses are compile-time offsets)
//      into a second shared tile;
//   3. column pass: each thread owns 2 adjacent columns x 8 rows and accumulates two FFMAs per
//      column pair (fma2_rn; a column pair is a natural 64-bit register pair), then streams out
//      with 8-byte stores.
// The taps stay in registers for a whole strip.  HBM traffic: 4 B read + 4 B written per element
// (24 B per RGB pixel) plus halo re-reads that hit in L2; the eager reference moves >= 32 B per
// element (two padded copies, two conv passes).  Tap order (ascending, FMA) is the generic kernel's,
// so the two agree bit for bit.
#pragma once
#include "tile_feed.cuh"

namespace kb200 {

constexpr int SEPT_TW = 128;
constexpr int SEPT_TH = 32;
constexpr int SEPT_XPAD = 8;                      // box starts 8 texels left of the tile: keeps the TMA start 16-B aligned
constexpr int SEPT_BW = SEPT_TW + 2 * SEPT_XPAD;  // 144

struct SepTiledParams {
  const float* kx;  // (Bkx, K)
  const float* ky;  // (Bky, K)
  float* out;
  int C, H, W, Bkx, Bky, planes;
  const float* x;   // LERP only: the input again (the epilogue re-reads the centre texels, an L2 hit)
  float lerp_w;     // LERP only: out = lerp(filtered, x, lerp_w)
};

// torch.lerp(start, end, w) as ATen evaluates it (ATen/native/Lerp.h): start + w * (end - start) for |w| < 0.5,
// end - (end - start) * (1 - w) otherwise; products feeding an add may contract to an FMA there, as here.
__device__ __forceinline__ float lerp_like_torch(float start, float end, float w) {
  const float diff = __fsub_rn(end, start);
  return fabsf(w) < 0.5f ? fmaf(w, diff, start) : fmaf(-diff, __fsub_rn(1.f, w), end);
}

template <int K>
constexpr size_t sept_smem_bytes() {  // two boxes, the row-filtered tile, two mbarriers
  return (size_t)(2 * (SEPT_TH + K - 1) * SEPT_BW + (SEPT_TH + K - 1) * SEPT_TW) * 4 + 2 * sizeof(uint64_t);
}

// LERP: the epilogue blends the filtered value with the input, out = lerp(filtered, x, w) -- unsharp_mask
// (filters/unsharp.py:53-54: gaussian_blur2d, then a separate torch.lerp pass over three full-size tensors) in the
// blur's own pass.
template <int K, int BORDER, bool LERP = false>
__global__ void __launch_bounds__(256, 3) sepfilter_tiled_kernel(const __grid_constant__ CUtensorMap tmap,
                                                                 const __grid_constant__ SepTiledParams p) {
  constexpr int HALO = (K - 1) / 2;
  static_assert(K % 2 == 1 && HALO <= SEPT_XPAD, "odd kernels up to 17 taps");
  constexpr int BH = SEPT_TH + K - 1;
  constexpr int BW = SEPT_BW;
  constexpr int TW = SEPT_TW, TH = SEPT_TH;
  constexpr int COL0 = SEPT_XPAD - HALO;        // box column of the first tap of output x = 0
  constexpr int A0 = COL0 & 3;                  // its offset inside an aligned float4
  constexpr int NV = (A0 + 4 + K - 1 + 3) / 4;  // aligned float4 loads that cover the 4-output window
  constexpr int TILE_FLOATS = BH * BW;
  constexpr uint32_t TILE_BYTES = TILE_FLOATS * 4;
  constexpr int ROW_ITERS = (BH + 7) / 8;       // 32 quads per row, 8 rows per sweep of the CTA
  constexpr int RY = 8;
  static_assert((TW / 2) * (TH / RY) == 256 && TW / 4 == 32, "thread mapping");

  extern __shared__ __align__(128) unsigned char sept_smem[];  // sept_smem_bytes<K>()
  float* tiles = reinterpret_cast<float*>(sept_smem);  // [2][BH][BW]
  float* mid = tiles + 2 * TILE_FLOATS;                // [BH][TW]
  uint64_t* full = reinterpret_cast<uint64_t*>(mid + BH * TW);  // [2]

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

  // thread roles (fixed for the whole kernel)
  const int rq = tid & 31, rr = tid >> 5;      // row pass: quad rq of rows rr, rr+8, ...
  const int cp = tid & 63, yb = tid >> 6;      // column pass: column pair cp, rows yb*8 .. yb*8+7

  int n = 0, strip, tx0, tx1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, tx0, tx1, cursor); ++seg) {
    const int plane = strip / tiles_y, ty = strip - plane * tiles_y;
    const int b = plane / p.C;
    const int y0 = ty * TH;
    // taps of this sample (filter.py:131,141-142: kernel index b mod Bk) stay in registers for the strip
    float kx[K];
    float2 ky2[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
      kx[j] = __ldg(p.kx + (size_t)(b % p.Bkx) * K + j);
      const float t = __ldg(p.ky + (size_t)(b % p.Bky) * K + j);
      ky2[j] = make_float2(t, t);
    }
    float* orow = p.out + (size_t)plane * p.H * p.W + (size_t)(y0 + yb * RY) * p.W + (size_t)tx0 * TW + 2 * cp;
    const bool rows_full = y0 + TH <= p.H;

    for (int tx = tx0; tx < tx1; ++tx, ++n, orow += TW) {
      const int s = n & 1;
      float* tile = tiles + s * TILE_FLOATS;
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      patch_box_border<BORDER>(tile, BH, BW, tx * TW - SEPT_XPAD, y0 - HALO, p);

      // ------------------------------------------------------------ row pass: tile -> mid
      {
        const float4* src4 = reinterpret_cast<const float4*>(tile + rr * BW + (COL0 & ~3) + 4 * rq);
        float4* dst4 = reinterpret_cast<float4*>(mid + rr * TW + 4 * rq);
#pragma unroll
        for (int it = 0; it < ROW_ITERS; ++it) {
          if ((it + 1) * 8 <= BH || rr + it * 8 < BH) {
            float win[NV * 4];
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              const float4 t = src4[it * 8 * (BW / 4) + v];
              win[4 * v] = t.x; win[4 * v + 1] = t.y; win[4 * v + 2] = t.z; win[4 * v + 3] = t.w;
            }
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int j = 0; j < K; ++j) {
#pragma unroll
              for (int o = 0; o < 4; ++o) acc[o] = __fmaf_rn(kx[j], win[A0 + o + j], acc[o]);
            }
            dst4[it * 8 * (TW / 4)] = make_float4(acc[0], acc[1], acc[2], acc[3]);
          }
        }
      }
      __syncthreads();  // mid complete, tile[s] no longer needed
      if (tid == 0) feed.issue(load);

      // ------------------------------------------------------------ column pass: mid -> out
      {
        float2 acc[RY];
#pragma unroll
        for (int o = 0; o < RY; ++o) acc[o] = make_float2(0.f, 0.f);
        const float2* m2 = reinterpret_cast<const float2*>(mid + (yb * RY) * TW + 2 * cp);
#pragma unroll
        for (int i = 0; i < RY + K - 1; ++i) {
          const float2 v = m2[i * (TW / 2)];
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            if (i - o >= 0 && i - o < K) acc[o] = fma2_rn(ky2[i - o], v, acc[o]);
          }
        }
        if (LERP) {
          const float* xin = p.x + (orow - p.out);
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            if (y0 + yb * RY + o < p.H && tx * TW + 2 * cp < p.W) {
              const float2 v = __ldg(reinterpret_cast<const float2*>(xin + (size_t)o * p.W));
              acc[o] = make_float2(lerp_like_torch(acc[o].x, v.x, p.lerp_w), lerp_like_torch(acc[o].y, v.y, p.lerp_w));
            }
          }
        }
        if (rows_full && (tx + 1) * TW <= p.W) {
          float* op = orow;
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            __stcs(reinterpret_cast<float2*>(op), acc[o]);
            op += p.W;
          }
        } else if (tx * TW + 2 * cp < p.W) {
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            if (y0 + yb * RY + o < p.H) __stcs(reinterpret_cast<float2*>(orow + (size_t)o * p.W), acc[o]);
          }
        }
      }
      __syncthreads();  // mid free for the next tile
    }
  }
}

// lerp_w == nullptr: plain filter; otherwise out = lerp(filtered, x, *lerp_w) (odd K <= 11 only)
int sepfilter_tiled_forward(const float* x, const float* kx, const float* ky, float* out, int B, int C, int H, int W, int Bkx, int kw,
                            int Bky, int kh, int border, int same, cudaStream_t st, const float* lerp_w = nullptr);

}  // namespace kb200
