// tools/hostemu reference (NOT product code): round 1's gather-per-tile SSIM kernel, verified on hardware then, kept as the
// bit-exact reference the emulator runs ssim_vwalk_kernel (the shipped kernel) against.
//
// kornia_b200 -- SSIM index map in one pass (fp32, odd Gaussian window K <= 11, 'reflect' border).
//
// The reference (kornia/metrics/ssim.py:92-139) runs filter2d_separable five times -- on img1, img2,
// img1^2, img2^2 and img1*img2, each call two F.pad copies and two grouped convolutions -- plus three
// product kernels and fourteen elementwise kernels for the index itself: > 250 B of HBM traffic per
// element.  Here one CTA produces a 64 x 32 tile of the map from the two input tiles:
//   1. the (64+K-1) x (32+K-1) boxes of both images are gathered into shared memory, the 'reflect'
//      border folded into the global index (no padded copy);
//   2. row pass: a thread owns 4 neighbouring outputs of a row, streams the 4+K-1 window positions once,
//      forms x, y, x*x, y*y, x*y (products rounded on their own, like the reference's img**2 / img1*img2
//      kernels) and accumulates the five row sums (5*K FMAs per output) into five shared planes;
//   3. column pass: a thread owns 2 columns x 4 rows and accumulates the five column sums with
//      two FMAs per column pair, then evaluates the index with one IEEE rounding per reference op and
//      stores it.
// HBM traffic: 8 B read + 4 B written per element.  The kernel is FMA bound (about 5*K*(1+(32+K-1)/32)
// FMAs per element: 127 for K = 11), not HBM bound.  Tap order (ascending, FMA) is that of the
// separable kernels, so the fused map equals the composition of this library's own filter2d_separable
// with torch's elementwise ops.
#pragma once
#include "../../kornia_b200/csrc/filter_generic.cuh"

namespace kb200 {

constexpr int SSIM_TW = 64;
constexpr int SSIM_TH = 32;
constexpr int SSIM_BW = SSIM_TW + 16;  // row stride of the input tiles: room for whole float4 windows

struct SsimParams {
  const float* a;     // img1 (planes,H,W)
  const float* b;     // img2
  const float* taps;  // (K,) device
  float* out;         // (planes,H,W)
  int planes, H, W;
  int tiles_x, tiles_y;
  int pair_ok;        // W even and out 8-byte aligned: float2 stores allowed
  float C1, C2, eps;
};

template <int K>
constexpr size_t ssim_smem_bytes() {
  return (size_t)(2 * (SSIM_TH + K - 1) * SSIM_BW + 5 * (SSIM_TH + K - 1) * SSIM_TW) * sizeof(float);
}

template <int K>
__global__ void __launch_bounds__(256, 2) ssim_tiled_kernel(const __grid_constant__ SsimParams p) {
  static_assert(K % 2 == 1 && K <= SSIM_MAX_K, "odd windows up to 11 taps");
  constexpr int HALO = K / 2;
  constexpr int TW = SSIM_TW, TH = SSIM_TH, BW = SSIM_BW;
  constexpr int BH = TH + K - 1;      // rows of the input box
  constexpr int BWV = TW + K - 1;     // valid columns of the input box
  constexpr int WIN = 4 + K - 1;      // window positions feeding 4 neighbouring outputs
  constexpr int NV = (WIN + 3) / 4;   // float4 loads per window
  constexpr int RY = 4;               // rows per thread in the column pass
  static_assert(4 * (TW / 4 - 1) + 4 * NV <= BW, "window loads stay inside a tile row");
  static_assert((TW / 2) * (TH / RY) == 256, "column-pass thread mapping");

  extern __shared__ __align__(16) float ssim_smem[];
  float* ta = ssim_smem;           // [BH][BW]
  float* tb = ta + BH * BW;        // [BH][BW]
  float* mid = tb + BH * BW;       // [5][BH][TW]

  const int tid = threadIdx.x;
  long long t = blockIdx.x;
  const int tx = (int)(t % p.tiles_x);
  t /= p.tiles_x;
  const int ty = (int)(t % p.tiles_y);
  const int plane = (int)(t / p.tiles_y);
  const int x0 = tx * TW, y0 = ty * TH;
  const size_t base = (size_t)plane * p.H * p.W;

  float k[K];
#pragma unroll
  for (int j = 0; j < K; ++j) k[j] = __ldg(p.taps + j);

  // ---------------------------------------------------------------- gather both boxes, border folded in
  for (int e = tid; e < BH * BWV; e += 256) {
    const int r = e / BWV, c = e - r * BWV;
    int gy = border_index<KB200_REFLECT>(y0 - HALO + r, p.H);
    int gx = border_index<KB200_REFLECT>(x0 - HALO + c, p.W);
    // cells beyond the padded image (partial edge tiles) feed only outputs that are never stored
    gy = min(max(gy, 0), p.H - 1);
    gx = min(max(gx, 0), p.W - 1);
    const size_t g = base + (size_t)gy * p.W + gx;
    ta[r * BW + c] = __ldg(p.a + g);
    tb[r * BW + c] = __ldg(p.b + g);
  }
  __syncthreads();

  // ---------------------------------------------------------------- row pass: 5 row sums -> mid
  for (int item = tid; item < BH * (TW / 4); item += 256) {
    const int r = item / (TW / 4), q = item - r * (TW / 4);
    const float4* pa = reinterpret_cast<const float4*>(ta + r * BW + 4 * q);
    const float4* pb = reinterpret_cast<const float4*>(tb + r * BW + 4 * q);
    float wa[NV * 4], wb[NV * 4];
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const float4 fa = pa[v], fb = pb[v];
      wa[4 * v] = fa.x; wa[4 * v + 1] = fa.y; wa[4 * v + 2] = fa.z; wa[4 * v + 3] = fa.w;
      wb[4 * v] = fb.x; wb[4 * v + 1] = fb.y; wb[4 * v + 2] = fb.z; wb[4 * v + 3] = fb.w;
    }
    float acc[5][4];
#pragma unroll
    for (int s = 0; s < 5; ++s)
#pragma unroll
      for (int o = 0; o < 4; ++o) acc[s][o] = 0.f;
#pragma unroll
    for (int w = 0; w < WIN; ++w) {
      const float x = wa[w], y = wb[w];
      const float v[5] = {x, y, __fmul_rn(x, x), __fmul_rn(y, y), __fmul_rn(x, y)};
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        if (w - o >= 0 && w - o < K) {
#pragma unroll
          for (int s = 0; s < 5; ++s) acc[s][o] = __fmaf_rn(k[w - o], v[s], acc[s][o]);
        }
      }
    }
#pragma unroll
    for (int s = 0; s < 5; ++s)
      *reinterpret_cast<float4*>(mid + (s * BH + r) * TW + 4 * q) = make_float4(acc[s][0], acc[s][1], acc[s][2], acc[s][3]);
  }
  __syncthreads();

  // ---------------------------------------------------------------- column pass + index
  const int cp = tid & 31, rg = tid >> 5;
  float2 acc[5][RY];
#pragma unroll
  for (int s = 0; s < 5; ++s)
#pragma unroll
    for (int o = 0; o < RY; ++o) acc[s][o] = make_float2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < RY + K - 1; ++i) {
#pragma unroll
    for (int s = 0; s < 5; ++s) {
      const float2 v = *reinterpret_cast<const float2*>(mid + (s * BH + rg * RY + i) * TW + 2 * cp);
#pragma unroll
      for (int o = 0; o < RY; ++o) {
        if (i - o >= 0 && i - o < K) acc[s][o] = __ffma2_rn(make_float2(k[i - o], k[i - o]), v, acc[s][o]);
      }
    }
  }

  const int gx = x0 + 2 * cp;
  if (gx >= p.W) return;
#pragma unroll
  for (int o = 0; o < RY; ++o) {
    const int gy = y0 + rg * RY + o;
    if (gy >= p.H) break;
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
    float* op = p.out + base + (size_t)gy * p.W + gx;
    if (p.pair_ok) {
      __stcs(reinterpret_cast<float2*>(op), make_float2(res[0], res[1]));
    } else {
      __stcs(op, res[0]);
      if (gx + 1 < p.W) __stcs(op + 1, res[1]);
    }
  }
}

int ssim_tiled_forward(const float* a, const float* b, const float* taps, float* out, int planes, int H, int W, int K, float C1,
                       float C2, float eps, cudaStream_t st);
// The library's SSIM kernel (ssim_vwalk.cuh, band-walking with TMA); KB200_EUNSUPPORTED outside its envelope.
int ssim_vwalk_forward(const float* a, const float* b, const float* taps, float* out, int planes, int H, int W, int K, float C1, float C2,
                       float eps, cudaStream_t st);

}  // namespace kb200
