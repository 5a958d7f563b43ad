// kornia_b200 -- separable K x K filter, one pass over HBM, walking DOWN column bands (fp32, 'same' padding).
//
// Same arithmetic as sepfilter_tiled_kernel (sepfilter_tiled.cuh: row pass with a register sliding window, column pass
// on column pairs (two FFMAs per pair), ascending tap order -- bit-identical results) with a different walk.  There a CTA
// moves left to right along a strip of 128 x 32 tiles and every tile row-filters its own 32 + K - 1 input rows: the
// K - 1 halo rows are filtered twice (by the tile above and the tile below), and with 8 rows per sweep of the CTA the
// 42 rows of the K = 11 blur take 6 sweeps, the last one three quarters idle -- the row pass costs 1.5x its useful work
// (ncu: FFMA 40 % of all instructions, the kernel is issue bound at 74 % of the HBM roofline, DESIGN.md 4.4).
// Here a CTA walks a 128-column band top to bottom and keeps the last K - 1 row-filtered rows in shared memory:
//   * per tile the TMA box is (128+16) x 32 rows (not 32 + K - 1), the row pass is exactly 4 full sweeps;
//   * the band (or band segment) starts with a (128+16) x (K-1) prologue box that seeds the carried rows;
//   * after the column pass the last K - 1 rows of the row-filtered tile move to the top of the buffer -- each
//     (row, quad) by the thread that overwrites it in the next row pass, so no extra barrier is needed;
//   * the vertical border (reflect / replicate) is applied to the row-filtered rows: row filtering acts along x and
//     the fold along y only selects a row, so fold-then-filter == filter-then-fold, bit for bit; the horizontal
//     border is patched in the box, on the two edge bands only and only over the out-of-image columns.
// Expected (not measured): ~18 % fewer issued instructions and 24 % less TMA / shared-memory fill traffic per tile.
//
// Selected by the sep_vwalk switch (sepfilter_vwalk.cu); tests/test_variants_gpu.py compares it bit for bit with
// sepfilter_tiled_kernel.
#pragma once
#include "sepfilter_tiled.cuh"

namespace kb200 {

// LERP: out = lerp(filtered, x, w) in the epilogue (unsharp_mask), as in sepfilter_tiled_kernel<K, BORDER, true>.
template <int K, int BORDER, bool LERP = false>
__global__ void __launch_bounds__(256, 3) sepfilter_vwalk_kernel(const __grid_constant__ CUtensorMap tmap_main,
                                                                 const __grid_constant__ CUtensorMap tmap_pro,
                                                                 const __grid_constant__ SepTiledParams p) {
  constexpr int HALO = (K - 1) / 2;
  constexpr int CARRY = K - 1;                  // row-filtered rows kept from one tile to the next
  static_assert(K % 2 == 1 && HALO <= SEPT_XPAD && CARRY <= SEPT_TH, "odd kernels up to 17 taps");
  constexpr int TW = SEPT_TW, TH = SEPT_TH, BW = SEPT_BW;
  constexpr int MH = TH + CARRY;                // rows of the row-filtered buffer: image rows t*TH - HALO ... + MH
  constexpr int COL0 = SEPT_XPAD - HALO;
  constexpr int A0 = COL0 & 3;
  constexpr int NV = (A0 + 4 + K - 1 + 3) / 4;
  constexpr int TILE_FLOATS = TH * BW;
  constexpr uint32_t TILE_BYTES = TILE_FLOATS * 4, PRO_BYTES = CARRY * BW * 4;
  constexpr int RY = 8;
  static_assert((TW / 2) * (TH / RY) == 256 && TW / 4 == 32 && TH == 32, "thread mapping");

  extern __shared__ __align__(128) unsigned char sepv_smem[];
  float* tiles = reinterpret_cast<float*>(sepv_smem);           // [2][TH][BW]; a prologue box uses the first CARRY rows of a slot
  float* mid = tiles + 2 * TILE_FLOATS;                         // [MH][TW]
  uint64_t* full = reinterpret_cast<uint64_t*>(mid + MH * TW);  // [2]

  const int tid = threadIdx.x;
  if (tid == 0) {
    tma::mbar_init(&full[0], 1);
    tma::mbar_init(&full[1], 1);
    tma::fence_barrier_init();
  }
  __syncthreads();

  const int bands = ceil_div(p.W, TW), tiles_y = ceil_div(p.H, TH);
  const Segments segs(p.planes * bands, tiles_y);  // a "strip" is a column band of one plane, walked top to bottom

  // The issuing thread walks the same box sequence as the CTA, two boxes ahead.  Per segment [t0, t1) of a band the
  // sequence is: prologue (t = t0 - 1), tile t0, ..., tile t1 - 1.
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
    tma::fence_proxy_async();
    if (ah.t < ah.t0) {  // prologue: image rows t0*TH - HALO ... + CARRY
      tma::mbar_arrive_expect_tx(&full[s], PRO_BYTES);
      tma::load_3d(tiles + s * TILE_FLOATS, &tmap_pro, &full[s], band * TW - SEPT_XPAD, ah.t0 * TH - HALO, plane);
    } else {             // tile t: image rows t*TH + HALO ... + TH (the rows below the carried ones)
      tma::mbar_arrive_expect_tx(&full[s], TILE_BYTES);
      tma::load_3d(tiles + s * TILE_FLOATS, &tmap_main, &full[s], band * TW - SEPT_XPAD, ah.t * TH + HALO, plane);
    }
    ahead_next();
  };
  if (tid == 0) {
    ahead_next();
    issue();
    issue();
  }

  const int rq = tid & 31, rr = tid >> 5;      // row pass: quad rq of box rows rr, rr+8, rr+16, rr+24
  const int cp = tid & 63, yb = tid >> 6;      // column pass: column pair cp, rows yb*8 .. yb*8+7
  float4* mid4 = reinterpret_cast<float4*>(mid);

  int n = 0, strip, t0, t1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, t0, t1, cursor); ++seg) {
    const int plane = strip / bands, band = strip - plane * bands;
    const int b = plane / p.C;
    const int x0 = band * TW, ox = x0 - SEPT_XPAD;
    float kx[K];
    float2 ky2[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
      kx[j] = __ldg(p.kx + (size_t)(b % p.Bkx) * K + j);
      const float t = __ldg(p.ky + (size_t)(b % p.Bky) * K + j);
      ky2[j] = make_float2(t, t);
    }
    const int nl = ox < 0 ? -ox : 0;                      // box columns [0, nl) lie left of the image
    const int nr = ox + BW > p.W ? ox + BW - p.W : 0;     // box columns [BW - nr, BW) lie right of it
    const bool x_edge = BORDER != KB200_CONSTANT && (nl + nr) > 0;
    const bool cols_full = x0 + TW <= p.W;

    for (int t = t0 - 1; t < t1; ++t, ++n) {
      const int s = n & 1;
      float* tile = tiles + s * TILE_FLOATS;
      const bool pro = t < t0;
      const int rows = pro ? CARRY : TH;
      tma::mbar_wait(&full[s], (n >> 1) & 1);

      if (x_edge) {  // CTA-uniform: fold the out-of-image columns of this box onto in-image columns of the same row
        const int ncols = nl + nr;
        for (int e = tid; e < rows * ncols; e += 256) {
          const int r = e / ncols, k = e - r * ncols;
          const int c = k < nl ? k : BW - nr + (k - nl);
          const int sc = border_index<BORDER>(ox + c, p.W) - ox;
          // the folded source of every column an output of this band needs lies inside the box; columns further
          // out (only reachable through the alignment padding) are never read
          if ((unsigned)sc < (unsigned)BW) tile[r * BW + c] = tile[r * BW + sc];
        }
        __syncthreads();
      }

      // ------------------------------------------------------------ row pass: box rows -> mid rows [0, CARRY) or [CARRY, MH)
      {
        const float4* src4 = reinterpret_cast<const float4*>(tile + rr * BW + (COL0 & ~3) + 4 * rq);
        float4* dst4 = mid4 + ((pro ? 0 : CARRY) + rr) * (TW / 4) + rq;
#pragma unroll
        for (int it = 0; it < TH / 8; ++it) {
          if (rr + it * 8 < rows) {
            float win[NV * 4];
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              const float4 q = src4[it * 8 * (BW / 4) + v];
              win[4 * v] = q.x; win[4 * v + 1] = q.y; win[4 * v + 2] = q.z; win[4 * v + 3] = q.w;
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
      __syncthreads();  // rows written, box consumed
      if (tid == 0) issue();
      if (pro) continue;

      const int y0 = t * TH, gy0 = y0 - HALO;  // gy0: image row of mid row 0
      if (BORDER != KB200_CONSTANT && (gy0 < 0 || gy0 + MH > p.H)) {  // CTA-uniform: first / last tiles of the band
        for (int e = tid; e < MH * (TW / 4); e += 256) {
          const int mr = e >> 5, qd = e & 31;
          const int gy = gy0 + mr;
          if ((unsigned)gy < (unsigned)p.H) continue;
          const int sr = border_index<BORDER>(gy, p.H) - gy0;  // an in-image row: never written by this loop
          if ((unsigned)sr < (unsigned)MH) mid4[mr * (TW / 4) + qd] = mid4[sr * (TW / 4) + qd];
        }
        __syncthreads();
      }

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
        float* orow = p.out + (size_t)plane * p.H * p.W + (size_t)(y0 + yb * RY) * p.W + (size_t)x0 + 2 * cp;
        if (LERP) {
          const float* xin = p.x + (orow - p.out);
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            if (y0 + yb * RY + o < p.H && x0 + 2 * cp < p.W) {
              const float2 v = __ldg(reinterpret_cast<const float2*>(xin + (size_t)o * p.W));
              acc[o] = make_float2(lerp_like_torch(acc[o].x, v.x, p.lerp_w), lerp_like_torch(acc[o].y, v.y, p.lerp_w));
            }
          }
        }
        if (y0 + TH <= p.H && cols_full) {
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            __stcs(reinterpret_cast<float2*>(orow), acc[o]);
            orow += p.W;
          }
        } else if (x0 + 2 * cp < p.W) {
#pragma unroll
          for (int o = 0; o < RY; ++o) {
            if (y0 + yb * RY + o < p.H) __stcs(reinterpret_cast<float2*>(orow + (size_t)o * p.W), acc[o]);
          }
        }
      }
      __syncthreads();  // every read of mid is done
      if (t + 1 < t1) {
        // carry mid rows [TH, MH) -> [0, CARRY): thread (rq, rr) moves exactly the (row, quad) cells it overwrites in
        // the next row pass (mid row CARRY + rr + 8*it, quad rq), so that write needs no barrier; the moved rows are
        // read after the next row pass's barrier
#pragma unroll
        for (int it = 0; it < TH / 8; ++it) {
          const int R = CARRY + rr + 8 * it;
          if (R >= TH) mid4[(R - TH) * (TW / 4) + rq] = mid4[R * (TW / 4) + rq];
        }
      }
    }
  }
}

}  // namespace kb200
