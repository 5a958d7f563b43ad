// kornia_b200 -- Harris and Shi-Tomasi (GFTT) responses in one pass, walking DOWN column bands with a TMA pipeline (fp32).
//
// Replaces kornia/feature/responses.py:99-126 / :182-203: spatial_gradient (3x3 stencils, replicate border), dx^2, dy^2,
// dx*dy, three gaussian_blur2d((7,7), (1,1)) calls (reflect border) and 7 (Harris) or ~17 (GFTT) elementwise kernels.
// The skeleton is ssim_vwalk_kernel's (vwalk.cuh): persistent CTAs walk 64-column bands top to bottom, the input box of
// each 32-row tile arrives by TMA into a double-buffered slot, and the 6 row-filtered rows shared by vertically adjacent
// tiles are carried in shared memory (three planes).  Arithmetic, one rounding per reference op, bit-identical to the
// composition:
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
#include "vwalk.cuh"

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
  return (size_t)(2 * (VWALK_TH + 2) * VWALK_BW + 3 * (VWALK_TH + CORNER_K - 1) * VWALK_TW) * sizeof(float) + 2 * sizeof(uint64_t);
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
  constexpr int TW = VWALK_TW, TH = VWALK_TH, BW = VWALK_BW;
  constexpr int BH = TH + 2;                     // box rows: the tile's product rows and one stencil row on each side
  constexpr int MH = TH + CARRY;                 // rows of a row-filtered plane: image rows t*TH - HALO ... + MH
  constexpr int COL0 = VWALK_XPAD - HALO - 1;    // box column of the stencil window of product position 0
  static_assert((COL0 & 3) == 0, "aligned stencil window");
  constexpr int WIN = 4 + K - 1;                 // product positions feeding 4 neighbouring outputs
  constexpr int NV = (WIN + 2 + 3) / 4;          // aligned float4 loads per stencil row
  constexpr int SLOT_FLOATS = BH * BW;
  constexpr uint32_t TILE_BYTES = BH * BW * 4, PRO_BYTES = (CARRY + 2) * BW * 4;
  constexpr int QUADS = VWALK_QUADS, RPS = VWALK_RPS, SWEEPS = VWALK_SWEEPS, RY = VWALK_RY;
  static_assert(COL0 + 4 * (QUADS - 1) + 4 * NV <= BW, "window loads stay inside a box row");

  extern __shared__ __align__(128) unsigned char corner_smem[];
  float* slots = reinterpret_cast<float*>(corner_smem);             // [2][BH][BW]
  float* mid = slots + 2 * SLOT_FLOATS;                             // [3][MH][TW]
  uint64_t* full = reinterpret_cast<uint64_t*>(mid + 3 * MH * TW);  // [2]

  const int tid = threadIdx.x;
  feed_init(full);

  const int bands = ceil_div(p.W, TW), tiles_y = ceil_div(p.H, TH);
  const Segments segs(p.planes * bands, tiles_y);

  // box sequence of a band segment [t0, t1): prologue (t = t0 - 1), tile t0, ..., tile t1 - 1
  TileFeed<true> feed(segs);
  auto load = [&](int slot, int strip, int t, bool prologue) {
    const int plane = strip / bands, band = strip - plane * bands;
    tma::mbar_arrive_expect_tx(&full[slot], prologue ? PRO_BYTES : TILE_BYTES);
    tma::load_3d(slots + slot * SLOT_FLOATS, prologue ? &pro : &map, &full[slot], band * TW - VWALK_XPAD,
                 prologue ? (t + 1) * TH - HALO - 1 : t * TH + HALO - 1, plane);  // the prologue: rows above tile t + 1
  };
  if (tid == 0) feed.start(load);

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
    const int x0 = band * TW, ox = x0 - VWALK_XPAD;
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

      patch_box_border<KB200_REPLICATE>(box, rows + 2, BW, ox, oy, p);  // replicate border of the image

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
      if (tid == 0) feed.issue(load);
      if (pro) continue;

      const int y0 = t * TH, gy0 = y0 - HALO;  // gy0: image row of mid row 0
      vwalk_reflect_rows<3, K>(mid4, gy0, p.H);  // first / last tiles of the band

      // ------------------------------------------------------------ column pass + response
      {
        float2 acc[3][RY];
        vwalk_column_pass<3, K>(mid, g, cp, rg, acc);
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
      if (t + 1 < t1) vwalk_carry_rows<3, K>(mid4, rq, rr);
    }
  }
}

// host entry (corner_vwalk.cu).  KB200_EUNSUPPORTED outside the kernel's envelope (rows that are not a multiple of 4 floats,
// misaligned buffers): the Python layer then composes spatial_gradient, three blurs and torch elementwise ops.
int corner_vwalk_forward(const float* x, const double* stencil, const float* taps, float k, const float* kptr, const float* s4, float* out,
                         int planes, int C, int H, int W, int kind, cudaStream_t st);

}  // namespace kb200
