// kornia_b200 -- Harris and Shi-Tomasi (GFTT) responses in one pass, walking DOWN column bands with a TMA pipeline (fp32).
//
// Replaces kornia/feature/responses.py:99-126 / :182-203: spatial_gradient (3x3 stencils, replicate border), dx^2, dy^2,
// dx*dy, three gaussian_blur2d((7,7), (1,1)) calls (reflect border) and 7 (Harris) or ~17 (GFTT) elementwise kernels.
// The skeleton is ssim_vwalk_kernel's: persistent CTAs walk 64-column bands top to bottom, the input box of each 32-row
// tile arrives by TMA into a double-buffered slot, and the 6 row-filtered rows shared by vertically adjacent tiles are
// carried in shared memory (three planes).  Arithmetic, one rounding per reference op, bit-identical to the composition:
//   * dx, dy with grad_tiled_kernel's tap order (row-major, ascending, every 3x3 tap including the zeros, __fmaf_rn);
//   * the three products rounded once each; row sums with ascending FMA taps, column sums on column pairs (fma2_rn),
//     as sepfilter_tiled_kernel;
//   * the epilogue with __fmul_rn / __fsub_rn / __fadd_rn / __fsqrt_rn and torch.minimum's NaN rule, then * sigmas^4.
// The two borders compose and do not commute: the image has a REPLICATE border for the derivative, the product planes a
// REFLECT border for the blur.  So the box is patched with replicate cells, products are formed at in-image positions
// only, and out-of-image product columns (edge quads, in registers) and row-filtered rows (first / last tiles) are
// copies of their reflections.  The stencil needs one more input row on each side of a tile's product rows: every box
// is TH + 2 rows high, its first and last rows shared with the neighbouring tiles' boxes (they come from L2).
//
// Launched by corner_vwalk.cu; tests/test_responses_gpu.py checks it bit for bit against the composition.
#pragma once
#include "sepfilter_tiled.cuh"
#include "filter_generic.cuh"
#include "ssim_vwalk.cuh"

namespace kb200 {

enum ResponseKind { RESP_HARRIS = 0, RESP_GFTT = 1, RESP_HESSIAN = 2 };

constexpr int CORNER_K = 7;  // the reference's gaussian_blur2d(., (7, 7), (1.0, 1.0))

struct CornerParams {
  const float* taps;  // (CORNER_K,) device Gaussian taps, rows and columns
  const float* kptr;  // device fp32 Harris k overriding `k`, or null
  const float* s4;    // (planes / C,) device sigmas^4, or null
  float* out;         // (planes,H,W)
  int planes, C, H, W;
  float k;
  float st[2 * 9];  // [dx, dy][3][3] correlation taps
};

constexpr size_t corner_smem_bytes() {
  return (size_t)(2 * (SSIMV_TH + 2) * SSIMV_BW + 3 * (SSIMV_TH + CORNER_K - 1) * SSIMV_TW) * sizeof(float) + 2 * sizeof(uint64_t);
}

// torch.minimum: NaN in either operand propagates (fminf would drop it)
__device__ __forceinline__ float torch_min(float a, float b) { return a != a ? a : (b != b ? b : fminf(a, b)); }

template <int KIND>
__device__ __forceinline__ float corner_score(float dx2, float dy2, float dxy, float k) {
  // responses.py:117-121 (Harris) / :192-198 (GFTT), one rounding per torch op
  const float det = __fsub_rn(__fmul_rn(dx2, dy2), __fmul_rn(dxy, dxy));
  const float tr = __fadd_rn(dx2, dy2);
  const float tr2 = __fmul_rn(tr, tr);
  if (KIND == RESP_HARRIS) return __fsub_rn(det, __fmul_rn(k, tr2));
  const float s = __fsqrt_rn(fabsf(__fsub_rn(tr2, __fmul_rn(4.0f, det))));
  return torch_min(__fmul_rn(0.5f, __fadd_rn(tr, s)), __fmul_rn(0.5f, __fsub_rn(tr, s)));
}

template <int KIND>
__global__ void __launch_bounds__(256, 2) corner_vwalk_kernel(const __grid_constant__ CUtensorMap map, const __grid_constant__ CUtensorMap pro,
                                                              const __grid_constant__ CornerParams p) {
  static_assert(KIND == RESP_HARRIS || KIND == RESP_GFTT, "corner epilogues");
  constexpr int K = CORNER_K, HALO = K / 2, CARRY = K - 1;
  constexpr int TW = SSIMV_TW, TH = SSIMV_TH, BW = SSIMV_BW;
  constexpr int BH = TH + 2;                     // box rows: the tile's product rows and one stencil row on each side
  constexpr int MH = TH + CARRY;                 // rows of a row-filtered plane: image rows t*TH - HALO ... + MH
  constexpr int COL0 = SSIMV_XPAD - HALO - 1;    // box column of the stencil window of product position 0
  static_assert((COL0 & 3) == 0, "aligned stencil window");
  constexpr int WIN = 4 + K - 1;                 // product positions feeding 4 neighbouring outputs
  constexpr int NV = (WIN + 2 + 3) / 4;          // aligned float4 loads per stencil row
  constexpr int SLOT_FLOATS = BH * BW;
  constexpr uint32_t TILE_BYTES = BH * BW * 4, PRO_BYTES = (CARRY + 2) * BW * 4;
  constexpr int QUADS = TW / 4;                  // 16 quads per row
  constexpr int RPS = 256 / QUADS;               // 16 rows per sweep of the CTA
  constexpr int SWEEPS = TH / RPS;               // 2
  constexpr int RY = 4;                          // rows per thread in the column pass
  static_assert((TW / 2) * (TH / RY) == 256 && SWEEPS * RPS == TH && CARRY <= RPS, "thread mapping");
  static_assert(COL0 + 4 * (QUADS - 1) + 4 * NV <= BW, "window loads stay inside a box row");

  extern __shared__ __align__(128) unsigned char corner_smem[];
  float* slots = reinterpret_cast<float*>(corner_smem);             // [2][BH][BW]
  float* mid = slots + 2 * SLOT_FLOATS;                             // [3][MH][TW]
  uint64_t* full = reinterpret_cast<uint64_t*>(mid + 3 * MH * TW);  // [2]

  const int tid = threadIdx.x;
  if (tid == 0) {
    tma::mbar_init(&full[0], 1);
    tma::mbar_init(&full[1], 1);
    tma::fence_barrier_init();
  }
  __syncthreads();

  const int bands = ceil_div(p.W, TW), tiles_y = ceil_div(p.H, TH);
  const Segments segs(p.planes * bands, tiles_y);

  // box sequence of a band segment [t0, t1): prologue (t = t0 - 1), tile t0, ..., tile t1 - 1; issued two boxes ahead
  struct Ahead {
    int seg, strip, t0, t1, cursor, t, n;
    bool live;
  } ah{0, 0, 0, 0, 0, 0, 0, false};
  auto ahead_next = [&]() {
    if (ah.live && ah.t + 1 < ah.t1) {
      ++ah.t;
      ++ah.n;
      return;
    }
    const bool first = !ah.live && ah.n == 0 && ah.seg == 0;
    ah.live = segs.get(ah.seg, ah.strip, ah.t0, ah.t1, ah.cursor);
    ++ah.seg;
    ah.t = ah.t0 - 1;
    if (!first) ++ah.n;
  };
  auto issue = [&]() {
    if (!ah.live) return;
    const int plane = ah.strip / bands, band = ah.strip - plane * bands;
    const int s = ah.n & 1;
    float* slot = slots + s * SLOT_FLOATS;
    tma::fence_proxy_async();
    if (ah.t < ah.t0) {
      tma::mbar_arrive_expect_tx(&full[s], PRO_BYTES);
      tma::load_3d(slot, &pro, &full[s], band * TW - SSIMV_XPAD, ah.t0 * TH - HALO - 1, plane);
    } else {
      tma::mbar_arrive_expect_tx(&full[s], TILE_BYTES);
      tma::load_3d(slot, &map, &full[s], band * TW - SSIMV_XPAD, ah.t * TH + HALO - 1, plane);
    }
    ahead_next();
  };
  if (tid == 0) {
    ahead_next();
    issue();
    issue();
  }

  float g[K];
#pragma unroll
  for (int j = 0; j < K; ++j) g[j] = __ldg(p.taps + j);
  const float kv = KIND == RESP_HARRIS && p.kptr ? __ldg(p.kptr) : p.k;

  const int rq = tid & (QUADS - 1), rr = tid / QUADS;  // row pass: quad rq of product rows rr, rr + 16
  const int cp = tid & 31, rg = tid >> 5;              // column pass: column pair cp, rows rg*4 .. rg*4+3
  float4* mid4 = reinterpret_cast<float4*>(mid);

  int n = 0, strip, t0, t1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, t0, t1, cursor); ++seg) {
    const int plane = strip / bands, band = strip - plane * bands;
    const int x0 = band * TW, ox = x0 - SSIMV_XPAD;
    const size_t base = (size_t)plane * p.H * p.W;
    const float s4 = p.s4 ? __ldg(p.s4 + plane / p.C) : 1.0f;
    const int gq = x0 + 4 * rq;                                  // first output column of this thread's row-pass quad
    const bool left = gq == 0, right = gq == p.W - 4;            // quads whose product window crosses the image edge

    for (int t = t0 - 1; t < t1; ++t, ++n) {
      const int s = n & 1;
      float* box = slots + s * SLOT_FLOATS;
      const bool pro = t < t0;
      const int rows = pro ? CARRY : TH;                       // product rows of this box
      const int oy = pro ? t0 * TH - HALO - 1 : t * TH + HALO - 1;  // image row of box row 0
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      if (ox < 0 || ox + BW > p.W || oy < 0 || oy + rows + 2 > p.H) {  // CTA-uniform: replicate border of the image
        for (int e = tid; e < (rows + 2) * BW; e += 256) {
          const int r = e / BW, c = e - r * BW;
          const int gy = oy + r, gx = ox + c;
          if ((unsigned)gy < (unsigned)p.H && (unsigned)gx < (unsigned)p.W) continue;
          const int sr = border_index<KB200_REPLICATE>(gy, p.H) - oy, sc = border_index<KB200_REPLICATE>(gx, p.W) - ox;
          if ((unsigned)sr < (unsigned)(rows + 2) && (unsigned)sc < (unsigned)BW) box[e] = box[sr * BW + sc];
        }
        __syncthreads();
      }

      // ------------------------------------------------------------ row pass: dx, dy, products, three row sums
#pragma unroll
      for (int it = 0; it < SWEEPS; ++it) {
        const int r = rr + it * RPS;
        if (r < rows) {
          float win[3][NV * 4];  // stencil rows r .. r+2, box columns COL0 + 4 rq ...
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            const float4* src = reinterpret_cast<const float4*>(box + (r + i) * BW + COL0 + 4 * rq);
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              const float4 f = src[v];
              win[i][4 * v] = f.x; win[i][4 * v + 1] = f.y; win[i][4 * v + 2] = f.z; win[i][4 * v + 3] = f.w;
            }
          }
          float prod[3][WIN];  // dx^2, dy^2, dx*dy at image columns gq - HALO + w
#pragma unroll
          for (int w = 0; w < WIN; ++w) {
            float d[2] = {0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
              for (int j = 0; j < 3; ++j)
#pragma unroll
                for (int o = 0; o < 2; ++o) d[o] = __fmaf_rn(p.st[(o * 3 + i) * 3 + j], win[i][w + j], d[o]);
            prod[0][w] = __fmul_rn(d[0], d[0]);
            prod[1][w] = __fmul_rn(d[1], d[1]);
            prod[2][w] = __fmul_rn(d[0], d[1]);
          }
          // reflect border of the product planes: columns -3..-1 are columns 3..1, W..W+2 are W-2..W-4 (W > 3)
          if (left) {
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
              for (int w = 0; w < HALO; ++w) prod[q][w] = prod[q][2 * HALO - w];
          }
          if (right) {
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
              for (int w = WIN - HALO; w < WIN; ++w) prod[q][w] = prod[q][2 * (WIN - HALO - 1) - w];
          }
          float acc[3][4];
#pragma unroll
          for (int q = 0; q < 3; ++q)
#pragma unroll
            for (int o = 0; o < 4; ++o) acc[q][o] = 0.f;
#pragma unroll
          for (int w = 0; w < WIN; ++w)
#pragma unroll
            for (int o = 0; o < 4; ++o)
              if (w - o >= 0 && w - o < K)
#pragma unroll
                for (int q = 0; q < 3; ++q) acc[q][o] = __fmaf_rn(g[w - o], prod[q][w], acc[q][o]);
          const int mr = (pro ? 0 : CARRY) + r;
#pragma unroll
          for (int q = 0; q < 3; ++q) mid4[(q * MH + mr) * QUADS + rq] = make_float4(acc[q][0], acc[q][1], acc[q][2], acc[q][3]);
        }
      }
      __syncthreads();  // rows written, box consumed
      if (tid == 0) issue();
      if (pro) continue;

      const int y0 = t * TH, gy0 = y0 - HALO;  // gy0: image row of mid row 0
      if (gy0 < 0 || gy0 + MH > p.H) {         // CTA-uniform: first / last tiles of the band -- reflect row-filtered rows
        for (int e = tid; e < MH * QUADS; e += 256) {
          const int mr = e / QUADS, qd = e - mr * QUADS;
          const int gy = gy0 + mr;
          if ((unsigned)gy < (unsigned)p.H) continue;
          const int sr = border_index<KB200_REFLECT>(gy, p.H) - gy0;  // an in-image row: never written by this loop
          if ((unsigned)sr < (unsigned)MH) {
#pragma unroll
            for (int q = 0; q < 3; ++q) mid4[(q * MH + mr) * QUADS + qd] = mid4[(q * MH + sr) * QUADS + qd];
          }
        }
        __syncthreads();
      }

      // ------------------------------------------------------------ column pass + response
      {
        float2 acc[3][RY];
#pragma unroll
        for (int q = 0; q < 3; ++q)
#pragma unroll
          for (int o = 0; o < RY; ++o) acc[q][o] = make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < RY + K - 1; ++i) {
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            const float2 v = *reinterpret_cast<const float2*>(mid + (q * MH + rg * RY + i) * TW + 2 * cp);
#pragma unroll
            for (int o = 0; o < RY; ++o) {
              if (i - o >= 0 && i - o < K) acc[q][o] = fma2_rn(make_float2(g[i - o], g[i - o]), v, acc[q][o]);
            }
          }
        }
        const int gx = x0 + 2 * cp;
        if (gx < p.W) {  // W % 4 == 0: whole pairs
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            const int gy = y0 + rg * RY + o;
            if (gy < p.H) {
              float res[2] = {corner_score<KIND>(acc[0][o].x, acc[1][o].x, acc[2][o].x, kv),
                              corner_score<KIND>(acc[0][o].y, acc[1][o].y, acc[2][o].y, kv)};
              if (p.s4) {
                res[0] = __fmul_rn(res[0], s4);
                res[1] = __fmul_rn(res[1], s4);
              }
              __stcs(reinterpret_cast<float2*>(p.out + base + (size_t)gy * p.W + gx), make_float2(res[0], res[1]));
            }
          }
        }
      }
      __syncthreads();  // every read of mid is done
      if (t + 1 < t1) {
        // carry rows [TH, MH) -> [0, CARRY) of the three planes: thread (rq, rr) moves exactly the cells it overwrites in
        // the next row pass (mid row CARRY + rr + 16*it, quad rq)
#pragma unroll
        for (int it = 0; it < SWEEPS; ++it) {
          const int R = CARRY + rr + it * RPS;
          if (R >= TH) {
#pragma unroll
            for (int q = 0; q < 3; ++q) mid4[(q * MH + R - TH) * QUADS + rq] = mid4[(q * MH + R) * QUADS + rq];
          }
        }
      }
    }
  }
}

// host entry (corner_vwalk.cu).  KB200_EUNSUPPORTED outside the kernel's envelope (rows that are not a multiple of 4 floats,
// misaligned buffers): the Python layer then composes spatial_gradient, three blurs and torch elementwise ops.
int corner_vwalk_forward(const float* x, const double* stencil, const float* taps, float k, const float* kptr, const float* s4, float* out,
                         int planes, int C, int H, int W, int kind, cudaStream_t st);

}  // namespace kb200
