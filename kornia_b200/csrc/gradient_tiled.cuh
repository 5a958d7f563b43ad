// kornia_b200 -- image derivatives on the TMA tile loader (fp32, K in {3,5}, NOUT in {2,3}, replicate border).
//
// Same arithmetic as spatial_gradient_fwd (gradient.cuh: NOUT stencils per pixel from one window, taps as constant-bank
// operands, row-major ascending FMA order -- bit-identical), on the skeleton of filter2d_tiled_kernel: persistent CTAs
// walk strips of 128 x 32 tiles, the (128+16) x (32+K-1) input box is TMA-loaded into shared memory and double
// buffered, the replicate border (kornia/filters/sobel.py:66-68: F.pad(..., 'replicate')) is a patch of the box on edge
// tiles.  A thread produces 4 columns x R rows of every output plane from a (R+K-1)-row register window fed by aligned
// LDS.128 -- the L1-gather kernel it replaces re-reads every input row K times through L1 with tiny CTAs (measured
// 50-66 % of the HBM roofline, DESIGN.md 4.5).  The epilogue E writes the NOUT planes (GRAD_PLANES), or fuses sobel's
// sqrt(gx^2 + gy^2 + eps) (GRAD_MAG, sobel.py:158-167), or hessian_response's dxx*dyy - dxy^2 times the optional sigma^4
// of the sample (GRAD_HESS, kornia/feature/responses.py:272-280), one rounding per torch op.
//
// Selected by the tiled_gradient switch (gradient.cu).
#pragma once
#include "filter2d_tiled.cuh"
#include "gradient.cuh"

namespace kb200 {

enum GradEpilogue { GRAD_PLANES, GRAD_MAG, GRAD_HESS };

struct GradTiledParams {
  float* out;  // (planes,NOUT,H,W), or (planes,H,W) for the magnitude and the Hessian response
  int H, W, planes;
  float eps;
  float taps[GRAD_MAX_OUT * GRAD_MAX_K * GRAD_MAX_K];  // [NOUT][K][K]
  const float* s4;  // GRAD_HESS: (planes / C,) sigmas^4, or null
  int C;
};

// resident CTAs per SM: three, except the 5x5 Hessian, which needs more than 80 registers to run without spills
template <int K, GradEpilogue E>
constexpr int grad_tiled_ctas() {
  return E == GRAD_HESS && K == 5 ? 2 : 3;
}

template <int K>
constexpr size_t grad_tiled_smem_bytes() {  // two boxes, two mbarriers
  return (size_t)(2 * (SEPT_TH + K - 1) * SEPT_BW) * 4 + 2 * sizeof(uint64_t);
}

template <int K, int NOUT, GradEpilogue E>
__global__ void __launch_bounds__(256, grad_tiled_ctas<K, E>()) grad_tiled_kernel(const __grid_constant__ CUtensorMap tmap,
                                                            const __grid_constant__ GradTiledParams p) {
  static_assert((K == 3 || K == 5) && NOUT >= 2 && NOUT <= GRAD_MAX_OUT && (E != GRAD_MAG || (NOUT == 2 && K == 3)) &&
                (E != GRAD_HESS || NOUT == 3), "stencil limits");
  constexpr int HALO = (K - 1) / 2;
  constexpr int TW = SEPT_TW, TH = SEPT_TH, BW = SEPT_BW;
  constexpr int BH = TH + K - 1;
  constexpr int COL0 = SEPT_XPAD - HALO;
  constexpr int A0 = COL0 & 3;
  constexpr int NV = (A0 + 4 + K - 1 + 3) / 4;
  constexpr int TILE_FLOATS = BH * BW;
  constexpr uint32_t TILE_BYTES = TILE_FLOATS * 4;
  constexpr int R = NOUT == 3 ? 2 : 4;      // output rows per thread and sweep
  constexpr int SWEEPS = TH / (8 * R);      // 8 row groups of R rows per sweep
  static_assert(TW / 4 == 32 && SWEEPS * 8 * R == TH, "thread mapping: 32 quads x 8 row groups x SWEEPS");

  extern __shared__ __align__(128) unsigned char gradt_smem[];  // grad_tiled_smem_bytes<K>()
  float* tiles = reinterpret_cast<float*>(gradt_smem);  // [2][BH][BW]
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

  const int q = tid & 31, rg = tid >> 5;  // quad q (columns 4q..4q+3), row group rg
  const size_t HW = (size_t)p.H * p.W;

  int n = 0, strip, tx0, tx1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, tx0, tx1, cursor); ++seg) {
    const int plane = strip / tiles_y, ty = strip - plane * tiles_y;
    const int y0 = ty * TH;
    float* oplane = p.out + (size_t)plane * (E == GRAD_PLANES ? NOUT : 1) * HW;
    const float s4 = E == GRAD_HESS && p.s4 ? __ldg(p.s4 + plane / p.C) : 1.0f;

    for (int tx = tx0; tx < tx1; ++tx, ++n) {
      const int s = n & 1;
      float* tile = tiles + s * TILE_FLOATS;
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      // replicate border: cells of the box outside the image copy the nearest image cell (which lies inside the box)
      patch_box_border<KB200_REPLICATE>(tile, BH, BW, tx * TW - SEPT_XPAD, y0 - HALO, p);

      const int gx0 = tx * TW + 4 * q;
#pragma unroll
      for (int sw = 0; sw < SWEEPS; ++sw) {
        const int row0 = (sw * 8 + rg) * R;  // first output row of this thread inside the tile
        float acc[NOUT][R][4];
#pragma unroll
        for (int o = 0; o < NOUT; ++o)
#pragma unroll
          for (int r = 0; r < R; ++r)
#pragma unroll
            for (int x = 0; x < 4; ++x) acc[o][r][x] = 0.f;
        const float4* src4 = reinterpret_cast<const float4*>(tile + row0 * BW + (COL0 & ~3) + 4 * q);
#pragma unroll
        for (int wr = 0; wr < R + K - 1; ++wr) {
          float win[NV * 4];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const float4 t = src4[wr * (BW / 4) + v];
            win[4 * v] = t.x; win[4 * v + 1] = t.y; win[4 * v + 2] = t.z; win[4 * v + 3] = t.w;
          }
          // window row wr is tap row i = wr - r of output row r: i ascends with wr for every output (row-major tap order)
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const int i = wr - r;
            if (i >= 0 && i < K) {
#pragma unroll
              for (int j = 0; j < K; ++j)
#pragma unroll
                for (int o = 0; o < NOUT; ++o) {
                  const float t = p.taps[(o * K + i) * K + j];
#pragma unroll
                  for (int x = 0; x < 4; ++x) acc[o][r][x] = __fmaf_rn(t, win[A0 + x + j], acc[o][r][x]);
                }
            }
          }
        }
        if (gx0 < p.W) {  // W % 4 == 0: whole quads
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const int gy = y0 + row0 + r;
            if (gy < p.H) {
              if (E == GRAD_MAG) {
                float m[4];
#pragma unroll
                for (int x = 0; x < 4; ++x)
                  m[x] = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(acc[0][r][x], acc[0][r][x]), __fmul_rn(acc[1][r][x], acc[1][r][x])), p.eps));
                __stcs(reinterpret_cast<float4*>(oplane + (size_t)gy * p.W + gx0), make_float4(m[0], m[1], m[2], m[3]));
              } else if (E == GRAD_HESS) {  // (dxx, dxy, dyy): dxx * dyy - dxy**2, then * sigmas.pow(4)
                float h[4];
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                  h[x] = __fsub_rn(__fmul_rn(acc[0][r][x], acc[2][r][x]), __fmul_rn(acc[1][r][x], acc[1][r][x]));
                  if (p.s4) h[x] = __fmul_rn(h[x], s4);
                }
                __stcs(reinterpret_cast<float4*>(oplane + (size_t)gy * p.W + gx0), make_float4(h[0], h[1], h[2], h[3]));
              } else {
#pragma unroll
                for (int o = 0; o < NOUT; ++o)
                  __stcs(reinterpret_cast<float4*>(oplane + (size_t)o * HW + (size_t)gy * p.W + gx0),
                         make_float4(acc[o][r][0], acc[o][r][1], acc[o][r][2], acc[o][r][3]));
              }
            }
          }
        }
      }
      __syncthreads();  // tile[s] consumed by every thread
      if (tid == 0) feed.issue(load);
    }
  }
}

// KB200_EUNSUPPORTED -> the caller runs spatial_gradient_fwd.
int spatial_gradient_tiled_forward(const float* x, const double* taps, float* out, int planes, int H, int W, int nout, int k, int magnitude,
                                   double eps, cudaStream_t st);
// hessian_response: taps (3,k,k) = (dxx, dxy, dyy), out (planes,H,W), s4 (planes / C,) or null.  KB200_EUNSUPPORTED -> the caller
// composes spatial_gradient and torch elementwise ops.
int hessian_tiled_forward(const float* x, const double* taps, const float* s4, float* out, int planes, int C, int H, int W, int k,
                          cudaStream_t st);

}  // namespace kb200
