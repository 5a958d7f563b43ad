// kornia_b200 -- SSIM index map in one pass, walking DOWN column bands with a TMA pipeline (fp32, odd K <= 11, reflect).
//
// Same arithmetic as ssim_tiled_kernel (ssim_tiled.cuh: products rounded on their own, five row sums with ascending
// FMA taps, five column sums on column pairs (two FFMAs per pair), the index with one rounding per reference op of
// kornia/metrics/ssim.py:92-139 -- bit-identical results), with persistent CTAs walking column bands.  The first version
// gathers both boxes with scalar loads, synchronises, row-filters 32 + K - 1 rows, synchronises, column-filters: one
// tile per CTA, nothing overlaps, measured 6.6 ms at B=64x3x1080x1920 (11 % of the HBM roofline, ~20 % of its FMA
// bound; DESIGN.md 4.5).  Here persistent CTAs walk 64-column bands top to bottom:
//   * both input boxes ((64+16) x 32) arrive by TMA into a double-buffered slot while the previous tile is filtered;
//   * the K - 1 row-filtered rows shared by vertically adjacent tiles are carried in shared memory (five planes), so
//     the row pass -- 5 K FMAs per element and the bulk of the work -- runs once per input row instead of
//     (32 + K - 1) / 32 times;
//   * the reflect border is a patch of the out-of-image box columns (edge bands only) and, vertically, a copy between
//     row-filtered rows (first / last tile of a band only).
//
// Launched by ssim_vwalk.cu; tests/test_variants_gpu.py checks it against the golden vectors, tools/hostemu bit for bit
// against the scalar form.
#pragma once
#include "vwalk.cuh"

namespace kb200 {

constexpr int SSIM_MAX_K = 11;  // odd Gaussian windows up to 11 taps (the reference's default window)

struct SsimVParams {
  const float* taps;  // (K,) device
  float* out;         // (planes,H,W)
  int planes, H, W;
  float C1, C2, eps;
};

template <int K>
constexpr size_t ssimv_smem_bytes() {
  return (size_t)(2 * 2 * VWALK_TH * VWALK_BW + 5 * (VWALK_TH + K - 1) * VWALK_TW) * sizeof(float) + 2 * sizeof(uint64_t);
}

template <int K>
__global__ void __launch_bounds__(256, 2) ssim_vwalk_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                                                            const __grid_constant__ CUtensorMap pro_a, const __grid_constant__ CUtensorMap pro_b,
                                                            const __grid_constant__ SsimVParams p) {
  static_assert(K % 2 == 1 && K >= 3 && K <= SSIM_MAX_K, "odd windows up to 11 taps");
  constexpr int HALO = K / 2, CARRY = K - 1;
  constexpr int TW = VWALK_TW, TH = VWALK_TH, BW = VWALK_BW;
  constexpr int MH = TH + CARRY;                 // rows of a row-filtered plane: image rows t*TH - HALO ... + MH
  constexpr int COL0 = VWALK_XPAD - HALO;        // box column of the first window position of output x = 0
  constexpr int A0 = COL0 & 3;
  constexpr int WIN = 4 + K - 1;                 // window positions feeding 4 neighbouring outputs
  constexpr int NV = (A0 + WIN + 3) / 4;         // aligned float4 loads per window
  constexpr int IMG_FLOATS = TH * BW;            // one image's box
  constexpr int SLOT_FLOATS = 2 * IMG_FLOATS;    // a slot holds the boxes of both images
  constexpr uint32_t TILE_BYTES = SLOT_FLOATS * 4, PRO_BYTES = 2 * CARRY * BW * 4;
  constexpr int QUADS = VWALK_QUADS, RPS = VWALK_RPS, SWEEPS = VWALK_SWEEPS, RY = VWALK_RY;
  static_assert((COL0 & ~3) + 4 * (QUADS - 1) + 4 * NV <= BW, "window loads stay inside a box row");

  extern __shared__ __align__(128) unsigned char ssimv_smem[];
  float* slots = reinterpret_cast<float*>(ssimv_smem);             // [2][2][TH][BW]
  float* mid = slots + 2 * SLOT_FLOATS;                            // [5][MH][TW]
  uint64_t* full = reinterpret_cast<uint64_t*>(mid + 5 * MH * TW);  // [2]

  const int tid = threadIdx.x;
  feed_init(full);

  const int bands = ceil_div(p.W, TW), tiles_y = ceil_div(p.H, TH);
  const Segments segs(p.planes * bands, tiles_y);

  // box sequence of a band segment [t0, t1): prologue (t = t0 - 1), tile t0, ..., tile t1 - 1
  TileFeed<true> feed(segs);
  auto load = [&](int slot, int strip, int t, bool prologue) {
    const int plane = strip / bands, band = strip - plane * bands;
    float* dst = slots + slot * SLOT_FLOATS;
    const int y = prologue ? (t + 1) * TH - HALO : t * TH + HALO;  // the prologue: the K - 1 rows above tile t + 1
    tma::mbar_arrive_expect_tx(&full[slot], prologue ? PRO_BYTES : TILE_BYTES);
    tma::load_3d(dst, prologue ? &pro_a : &map_a, &full[slot], band * TW - VWALK_XPAD, y, plane);
    tma::load_3d(dst + IMG_FLOATS, prologue ? &pro_b : &map_b, &full[slot], band * TW - VWALK_XPAD, y, plane);
  };
  if (tid == 0) feed.start(load);

  float k[K];
#pragma unroll
  for (int j = 0; j < K; ++j) k[j] = __ldg(p.taps + j);

  const int rq = tid & (QUADS - 1), rr = tid / QUADS;  // row pass: quad rq of box rows rr, rr + 16
  const int cp = tid & 31, rg = tid >> 5;              // column pass: column pair cp, rows rg*4 .. rg*4+3
  float4* mid4 = reinterpret_cast<float4*>(mid);

  int n = 0, strip, t0, t1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, t0, t1, cursor); ++seg) {
    const int plane = strip / bands, band = strip - plane * bands;
    const int x0 = band * TW, ox = x0 - VWALK_XPAD;
    const int nl = ox < 0 ? -ox : 0;                    // box columns [0, nl) lie left of the image
    const int nr = ox + BW > p.W ? ox + BW - p.W : 0;   // box columns [BW - nr, BW) lie right of it
    const size_t base = (size_t)plane * p.H * p.W;

    for (int t = t0 - 1; t < t1; ++t, ++n) {
      const int s = n & 1;
      float* ta = slots + s * SLOT_FLOATS;
      float* tb = ta + IMG_FLOATS;
      const bool pro = t < t0;
      const int rows = pro ? CARRY : TH;
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      if (nl + nr > 0) {  // CTA-uniform (edge bands): reflect the out-of-image columns of both boxes
        const int ncols = nl + nr;
        for (int e = tid; e < rows * ncols; e += 256) {
          const int r = e / ncols, kk = e - r * ncols;
          const int c = kk < nl ? kk : BW - nr + (kk - nl);
          const int sc = border_index<KB200_REFLECT>(ox + c, p.W) - ox;
          if ((unsigned)sc < (unsigned)BW) {
            ta[r * BW + c] = ta[r * BW + sc];
            tb[r * BW + c] = tb[r * BW + sc];
          }
        }
        __syncthreads();
      }

      // ------------------------------------------------------------ row pass: five row sums -> mid rows [0,CARRY) or [CARRY,MH)
#pragma unroll
      for (int it = 0; it < SWEEPS; ++it) {
        const int r = rr + it * RPS;
        if (r < rows) {
          const float4* pa = reinterpret_cast<const float4*>(ta + r * BW + (COL0 & ~3) + 4 * rq);
          const float4* pb = reinterpret_cast<const float4*>(tb + r * BW + (COL0 & ~3) + 4 * rq);
          float wa[NV * 4], wb[NV * 4];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const float4 fa = pa[v], fb = pb[v];
            wa[4 * v] = fa.x; wa[4 * v + 1] = fa.y; wa[4 * v + 2] = fa.z; wa[4 * v + 3] = fa.w;
            wb[4 * v] = fb.x; wb[4 * v + 1] = fb.y; wb[4 * v + 2] = fb.z; wb[4 * v + 3] = fb.w;
          }
          float acc[5][4];
#pragma unroll
          for (int q = 0; q < 5; ++q)
#pragma unroll
            for (int o = 0; o < 4; ++o) acc[q][o] = 0.f;
#pragma unroll
          for (int w = 0; w < WIN; ++w) {
            const float x = wa[A0 + w], y = wb[A0 + w];
            const float v[5] = {x, y, __fmul_rn(x, x), __fmul_rn(y, y), __fmul_rn(x, y)};
#pragma unroll
            for (int o = 0; o < 4; ++o) {
              if (w - o >= 0 && w - o < K) {
#pragma unroll
                for (int q = 0; q < 5; ++q) acc[q][o] = __fmaf_rn(k[w - o], v[q], acc[q][o]);
              }
            }
          }
          const int mr = (pro ? 0 : CARRY) + r;
#pragma unroll
          for (int q = 0; q < 5; ++q) mid4[(q * MH + mr) * QUADS + rq] = make_float4(acc[q][0], acc[q][1], acc[q][2], acc[q][3]);
        }
      }
      __syncthreads();  // rows written, boxes consumed
      if (tid == 0) feed.issue(load);
      if (pro) continue;

      const int y0 = t * TH, gy0 = y0 - HALO;  // gy0: image row of mid row 0
      vwalk_reflect_rows<5, K>(mid4, gy0, p.H);  // first / last tiles of the band

      // ------------------------------------------------------------ column pass + index
      {
        float2 acc[5][RY];
        vwalk_column_pass<5, K>(mid, k, cp, rg, acc);
        const int gx = x0 + 2 * cp;
        if (gx < p.W) {  // W % 4 == 0: whole pairs
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            const int gy = y0 + rg * RY + o;
            if (gy < p.H) {
              float res[2];
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float mu1 = h ? acc[0][o].y : acc[0][o].x, mu2 = h ? acc[1][o].y : acc[1][o].x;
                const float e11 = h ? acc[2][o].y : acc[2][o].x, e22 = h ? acc[3][o].y : acc[3][o].x;
                const float e12 = h ? acc[4][o].y : acc[4][o].x;
                // ssim.py:117-139, one rounding per torch op
                const float mu1_sq = __fmul_rn(mu1, mu1), mu2_sq = __fmul_rn(mu2, mu2), mu1_mu2 = __fmul_rn(mu1, mu2);
                const float sigma1_sq = __fsub_rn(e11, mu1_sq), sigma2_sq = __fsub_rn(e22, mu2_sq), sigma12 = __fsub_rn(e12, mu1_mu2);
                const float num = __fmul_rn(__fadd_rn(__fmul_rn(2.0f, mu1_mu2), p.C1), __fadd_rn(__fmul_rn(2.0f, sigma12), p.C2));
                const float den = __fmul_rn(__fadd_rn(__fadd_rn(mu1_sq, mu2_sq), p.C1), __fadd_rn(__fadd_rn(sigma1_sq, sigma2_sq), p.C2));
                res[h] = __fdiv_rn(num, __fadd_rn(den, p.eps));
              }
              __stcs(reinterpret_cast<float2*>(p.out + base + (size_t)gy * p.W + gx), make_float2(res[0], res[1]));
            }
          }
        }
      }
      __syncthreads();  // every read of mid is done
      if (t + 1 < t1) vwalk_carry_rows<5, K>(mid4, rq, rr);
    }
  }
}

// host entry (ssim_vwalk.cu).  KB200_EUNSUPPORTED outside the kernel's envelope (even / > 11-tap windows, rows that are not a
// multiple of 4 floats): the Python layer then composes five one-pass blurs and torch elementwise ops.
int ssim_vwalk_forward(const float* a, const float* b, const float* taps, float* out, int planes, int H, int W, int K, float C1, float C2,
                       float eps, cudaStream_t st);

}  // namespace kb200
