// kornia_b200 -- tiled fused warp backward, second structure: every warp is its own pipeline (fp32, bilinear,
// zeros/border, C = 3 or 1).
//
// Same per-pixel arithmetic as warp_bwd_tma (warp_bwd_tma.cuh: the coordinate chain of imgwarp.py:165-170 op for op,
// shared-reciprocal IEEE division, strip adds with LDS/FADD/STS flushed by one TMA reduce-add per warp and tile,
// d/dM partials in registers -> shuffle -> records -> fixed-order second stage), different synchronisation.
//
// warp_bwd_tma idles on the consumers' mbarrier spin.  That kernel has ONE shared stage (the 72x40xC source box + the
// per-warp strip origins published by warp 0), so every tile ends with
//     all warps -> `empty` -> warp 0 waits -> publishes + issues the box load -> box lands -> `full` -> all warps
// and the CTA idles through that chain; the fast warps of a tile wait for the slowest.
// Here nothing is shared between the warps of a CTA except the static tile schedule:
//   * a warp maps the four corners of ITS 64 x 4 sub-tile (lanes 0..3, replicated over the warp), derives its own
//     72 x 8 window origin and -- for d/dM -- TMA-loads that window of `src` (72 x 8 x C, 6.9 KB) into its own buffer
//     on its own mbarrier, while it zero-fills its accumulation strip and fetches the first upstream-gradient row;
//   * the window of the source taps and the window of the accumulation strip are the same rectangle, so the fast-path
//     test is one window test instead of two;
//   * no CTA-wide barrier or handshake inside the tile loop: 16 independent warps per SM hide each other's latency.
// Shared memory: 8 x (window + strip) = 110.6 KB per CTA with both gradients -> still 2 CTAs/SM.
//
// d/dsrc is bit-identical to the column-pair lanes up to the order of the TMA reduce-adds; stride-1 lanes (STRIDE1) are the default.
#pragma once
#include <type_traits>

#include "warp_bwd_tma.cuh"

namespace kb200 {

// STRIDE1: lane <-> column (x0 + lane, x0 + 32 + lane) instead of column pairs (2 lane, 2 lane + 1).  Stride-2 lanes make every
// strip / window access a 2-way bank conflict but never
// share a floor cell; stride-1 lanes are conflict-free but two neighbours fall into one cell wherever the map minifies.  The vote
// stays warp-uniform: no duplicate in the instruction -> the un-predicated tap code; duplicates of multiplicity 2 -> two
// predicated rounds (first-of-cell lanes, then second-of-cell lanes); deeper pile-ups -> the exact path.
//
// DYN: the work is not dealt out in advance.  The warps are independent pipelines already, so each WARP draws its next item -- one
// 4-row slice of a chunk of tiles of a strip -- from a counter in global memory; the eight slices of a chunk are consecutive items.
// No CTA-wide step is added.  The d/dM record of an item goes to row (chunk, slice), so the second stage sums the same partials in
// a fixed order whatever warp produced them: still deterministic.  (With a static deal the slowest SM is active
// much longer than the average.)
template <int NC, int PAD, bool PROJ, bool ALIGN, bool NEED_SRC, bool NEED_M, bool STRIDE1 = false, bool DYN = false>
__global__ void __launch_bounds__(BWD_THREADS, 2) warp_bwd_tma2(const __grid_constant__ CUtensorMap tmap_srcwin,
                                                                const __grid_constant__ CUtensorMap tmap_gsrc,
                                                                const __grid_constant__ CUtensorMap tmap_gout,
                                                                const __grid_constant__ TmaBwdParams p) {
  using R = RN<float>;
  constexpr int TW = 64, TH = 32, BW = 72;
  constexpr int NJ = TW / 32, RPW = TH / TMA_CONSUMER_WARPS;
  constexpr int SPLANE = BW * BWD_SH;               // one channel of a window / strip
  constexpr int STRIP_FLOATS = NC * SPLANE;
  constexpr uint32_t WIN_BYTES = STRIP_FLOATS * 4;
  static_assert((STRIP_FLOATS * 4) % 128 == 0, "per-warp buffers stay 128-byte aligned");

  extern __shared__ __align__(128) unsigned char bwd2_smem[];
  float* wins = reinterpret_cast<float*>(bwd2_smem);                                   // [8 warps][NC][SH][BW] (NEED_M only)
  float* strips = wins + (NEED_M ? TMA_CONSUMER_WARPS * STRIP_FLOATS : 0);              // [8 warps][NC][SH][BW] (NEED_SRC only)
  uint64_t* wfull = reinterpret_cast<uint64_t*>(strips + (NEED_SRC ? TMA_CONSUMER_WARPS * STRIP_FLOATS : 0));  // [8]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < TMA_CONSUMER_WARPS; ++i) tma::mbar_init(&wfull[i], 1);
    tma::fence_barrier_init();
    if (NEED_M) tma::prefetch_map(&tmap_srcwin);
  }
  if (NEED_M && !DYN) {  // mark every record row of this CTA unused; rows are claimed as segments are processed
    for (int i = threadIdx.x; i < p.max_segs; i += blockDim.x) p.record_batch[(size_t)blockIdx.x * p.max_segs + i] = -1;
  }
  __syncthreads();  // the only CTA-wide barrier of the kernel

  const int tiles_x = ceil_div(p.w, TW), tiles_y = ceil_div(p.h, TH);
  const Segments segs(p.B * tiles_y, tiles_x);
  const int H = p.H, W = p.W;
  const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1), Wf = (float)W, Hf = (float)H;
  const size_t oplane = (size_t)p.h * p.w;
  float* strip_mem = strips + warp * STRIP_FLOATS;
  float* win_mem = wins + warp * STRIP_FLOATS;
  const uint32_t strip_u32 = tma::smem_u32(strip_mem), win_u32 = tma::smem_u32(win_mem);
  uint64_t* my_full = &wfull[warp];
  uint32_t phase = 0;

  const int dyn_ch = DYN ? max(p.chunk_tiles, 1) : 1, dyn_cps = ceil_div(tiles_x, dyn_ch);
  const int dyn_items = DYN ? p.B * tiles_y * dyn_cps * TMA_CONSUMER_WARPS : 0;
  int seg_strip, tx0, tx1, cursor = 0;
  int drawn = 0;  // DYN: the item this warp drew ahead
  if (DYN && lane == 0) drawn = atomicAdd(p.counter, 1);
  for (int seg = 0;; ++seg) {
    int slice = warp;        // which 4-row slice of the tiles this warp takes
    int record_row = 0;      // row of the d/dM record of this run of tiles
    if (DYN) {
      const int item = __shfl_sync(0xffffffffu, drawn, 0);
      if (item >= dyn_items) break;
      if (lane == 0) drawn = atomicAdd(p.counter, 1);  // the next item: its round trip through L2 overlaps this one's tiles
      const int chunk = item / TMA_CONSUMER_WARPS;
      slice = item - chunk * TMA_CONSUMER_WARPS;
      seg_strip = chunk / dyn_cps;
      tx0 = (chunk - seg_strip * dyn_cps) * dyn_ch;
      tx1 = min(tiles_x, tx0 + dyn_ch);
      record_row = chunk;
    } else {
      if (!segs.get(seg, seg_strip, tx0, tx1, cursor)) break;
      record_row = blockIdx.x * p.max_segs + seg;
    }
    const int b = seg_strip / tiles_y, ty = seg_strip - b * tiles_y;
    Mat3<float> m;
    m.load(p.m + (p.Bm == 1 ? 0 : (size_t)b * 9));
    const int y_base = ty * TH + slice * RPW;
    const float* gbase = p.gout + (size_t)b * NC * oplane;
    float pm[9];  // d/dm partials of this thread over the whole segment
#pragma unroll
    for (int k = 0; k < 9; ++k) pm[k] = 0.f;
    const float ux_scale = ALIGN ? Wm1 * 0.5f : Wf * 0.5f, uy_scale = ALIGN ? Hm1 * 0.5f : Hf * 0.5f;

    for (int tx = tx0; tx < tx1; ++tx) {
      // ---------------------------------------------------------------- this warp's window (all lanes, replicated)
      int sox, soy;
      bool win_ok;
      {
        const int py = min(y_base + ((lane & 2) ? RPW - 1 : 0), p.h - 1);
        const int px = min(tx * TW + ((lane & 1) ? TW - 1 : 0), p.w - 1);
        float gx, gy, den;
        map_point<float, PROJ>(m, __ldg(p.bx + px), __ldg(p.by + py), gx, gy, den);
        float ix = unnorm<ALIGN>(gx, Wm1, Wf), iy = unnorm<ALIGN>(gy, Hm1, Hf);
        bool ok = fabsf(ix) < 4.0e6f && fabsf(iy) < 4.0e6f;
        if (PROJ) {  // lanes hold the four corners eight times over: the ballot is over the corners
          const unsigned neg = __ballot_sync(0xffffffffu, den < 0.f);
          ok = ok && (neg == 0u || neg == 0xffffffffu) && fabsf(den) > 1e-12f;
        }
        if (PAD == KB200_BORDER) {
          ix = clip_coord(ix, W);
          iy = clip_coord(iy, H);
        }
        float lo_x = ix, hi_x = ix, lo_y = iy;
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          lo_x = fminf(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o));
          hi_x = fmaxf(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
          lo_y = fminf(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o));
        }
        win_ok = __all_sync(0xffffffffu, ok);
        const int x_lo = (int)floorf(lo_x), x_hi = (int)floorf(hi_x) + 1;
        const int need_w = x_hi - x_lo + 1;
        const int spare = BW - need_w - 3;
        const int ox = (x_lo - (spare > 0 ? spare / 2 : 0)) & ~3;  // TMA: 16-byte aligned start
        // origins are clamped to the image: a TMA reduce cannot take negative coordinates, and taps left of / above
        // the image are out of bounds anyway (they take the exact path)
        sox = win_ok ? max(ox, 0) : 0x20000000;
        soy = win_ok ? max((int)floorf(lo_y), 0) : 0x20000000;
      }
      if (slice == 0 && tx + 1 < tx1 && tma::elect_one()) tma::prefetch_3d(&tmap_gout, (tx + 1) * TW, ty * TH, b * NC);
      __syncwarp();

      // lane <-> output columns (2 lane, 2 lane + 1): inside one instruction the lanes are two pixels apart, so
      // their floor cells are distinct whenever the source step per output pixel exceeds 1/2
      constexpr int JS = STRIDE1 ? 32 : 1;  // column distance of a lane's two pixels
      const int x0 = tx * TW + (STRIDE1 ? lane : 2 * lane);
      float bxv[NJ], cx0[NJ], cx1[NJ], cx2[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        bxv[j] = __ldg(p.bx + min(x0 + JS * j, p.w - 1));
        cx0[j] = R::mul(m.m00, bxv[j]);
        cx1[j] = R::mul(m.m10, bxv[j]);
        cx2[j] = PROJ ? R::mul(m.m20, bxv[j]) : 0.f;
      }
      if (NEED_M && win_ok) {
        // every lane has finished reading the previous tile's window (program order + the __syncwarp above)
        if (tma::elect_one()) {
          tma::fence_proxy_async();
          tma::mbar_arrive_expect_tx(my_full, WIN_BYTES);
          tma::load_3d(win_mem, &tmap_srcwin, my_full, sox, soy, b * NC);
        }
        __syncwarp();
      }
      if (NEED_SRC) {
        // the previous tile's strip must have been read by the TMA unit before it is cleared
        if (lane == 0) tma::bulk_wait_read0();
        __syncwarp();
        float4* z = reinterpret_cast<float4*>(strip_mem);
        for (int e = lane; e < STRIP_FLOATS / 4; e += 32) z[e] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      // cell (ly, lx) of the window / strip = (Y - MAGIC - soy, X - MAGIC - sox)
      const unsigned kwin = (unsigned)(FLOOR_MAGIC_BITS + soy) * (unsigned)BW + (unsigned)(FLOOR_MAGIC_BITS + sox);
      const uint32_t strip_base = strip_u32 - 4u * kwin, win_base = win_u32 - 4u * kwin;
      // A window that starts at the image edge also serves coordinates in [-1, 0) under 'zeros': the tap in column / row -1
      // is outside the image (no contribution, value 0) and is predicated off in the EDGE copy of the row loop below.  Before,
      // every pixel of such a tile -- one tile in ten at 720p -- took the per-pixel atomics path.
      const bool edge_x = PAD == KB200_ZEROS && sox == 0, edge_y = PAD == KB200_ZEROS && soy == 0;
      const float s_lo_x = edge_x ? -1.f : (float)sox, s_hi_x = (float)(sox + BW - 1);
      const float s_lo_y = edge_y ? -1.f : (float)soy, s_hi_y = (float)(soy + BWD_SH - 1);

      // upstream gradient, software-pipelined one row ahead: both columns of a lane in one 8-byte load per channel
      float2 go_next[NC];
      auto load_gout_row = [&](int yy, float2 (&dst)[NC]) {
        const float* g0 = gbase + (size_t)min(yy, p.h - 1) * p.w;
        if (STRIDE1) {  // two coalesced 128-byte rows per channel
          const int xa = min(x0, p.w - 1), xb = min(x0 + 32, p.w - 1);
#pragma unroll
          for (int c = 0; c < NC; ++c) dst[c] = make_float2(__ldg(g0 + c * oplane + xa), __ldg(g0 + c * oplane + xb));
        } else {        // both columns of a lane in one 8-byte load per channel
          const float* g = g0 + min(x0, p.w - 2);
#pragma unroll
          for (int c = 0; c < NC; ++c) dst[c] = __ldg(reinterpret_cast<const float2*>(g + c * oplane));
        }
      };
      load_gout_row(y_base, go_next);
      if (NEED_M && win_ok) {  // warp-uniform
        tma::mbar_wait(my_full, phase);
        phase ^= 1;
      }
      __syncwarp();  // strip cleared by all lanes

      auto rows = [&](auto edge_tag) {
      constexpr bool EDGE = decltype(edge_tag)::value;
#pragma unroll 1
      for (int i = 0; i < RPW; ++i) {
        const int y = y_base + i;
        const float byr = __ldg(p.by + min(y, p.h - 1));
        const float cy0 = R::mul(m.m01, byr), cy1 = R::mul(m.m11, byr), cy2 = PROJ ? R::mul(m.m21, byr) : 0.f;
        float2 go2[NC];
#pragma unroll
        for (int c = 0; c < NC; ++c) go2[c] = go_next[c];
        if (i + 1 < RPW) load_gout_row(y + 1, go_next);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int x = x0 + JS * j;
          const bool live = y < p.h && x < p.w;  // warp-uniform in y, not in x
          const float nx = R::add(R::add(cx0[j], cy0), m.m02);
          const float ny = R::add(R::add(cx1[j], cy1), m.m12);
          float gx = nx, gy = ny, rden = 1.f;
          bool den_ok = true;
          if (PROJ) {
            const float den = R::add(R::add(cx2[j], cy2), m.m22);
            den_ok = fabsf(den) >= 8.67361738e-19f;  // 2^-60: below it the shared-reciprocal division is not exact
            rden = refined_rcp(den);
            gx = div_by_rcp(nx, den, rden);
            gy = div_by_rcp(ny, den, rden);
            if (!den_ok) {  // rare: exact library division
              gx = __fdiv_rn(nx, den);
              gy = __fdiv_rn(ny, den);
              rden = __fdiv_rn(1.f, den);
            }
          }
          float ix = unnorm<ALIGN>(gx, Wm1, Wf), iy = unnorm<ALIGN>(gy, Hm1, Hf);
          float px = 1.f, py = 1.f;  // d(padded coordinate)/d(coordinate): 0 where the border clamp is active
          if (PAD == KB200_BORDER) {
            // pad_coord_grad's clamp (ATen's clip_coordinates_set_grad): comparisons, so a NaN coordinate stays NaN, takes the
            // exact path and scatters nothing -- fminf / fmaxf would turn it into texel 0
            if (ix <= 0.f) { ix = 0.f; px = 0.f; } else if (ix >= Wm1) { ix = Wm1; px = 0.f; }
            if (iy <= 0.f) { iy = 0.f; py = 0.f; } else if (iy >= Hm1) { iy = Hm1; py = 0.f; }
          }
          const float tX = __fadd_rd(ix, FLOOR_MAGIC), tY = __fadd_rd(iy, FLOOR_MAGIC);
          const int X = __float_as_int(tX), Y = __float_as_int(tY);
          // fast path (all lanes of the warp must agree): the four taps inside this warp's window, and no two lanes of
          // this instruction share a floor cell -- along a row the map is monotone, so duplicates are adjacent lanes
          bool ok = live && den_ok && ix >= s_lo_x && ix < s_hi_x && iy >= s_lo_y && iy < s_hi_y;
          const int Xl = __shfl_up_sync(0xffffffffu, X, 1), Yl = __shfl_up_sync(0xffffffffu, Y, 1);
          const bool same1 = lane > 0 && Xl == X && Yl == Y;  // second (or later) lane of its floor cell
          bool two_rounds = false;
          if (STRIDE1) {
            const bool same2 = __shfl_up_sync(0xffffffffu, same1 ? 1 : 0, 1) != 0 && same1;  // third or later: exact path
            if (same2) ok = false;
            two_rounds = NEED_SRC && __any_sync(0xffffffffu, same1);
          } else if (same1) {
            ok = false;
          }
          float gix = 0.f, giy = 0.f;
          if (__all_sync(0xffffffffu, ok)) {
            const float x0f = R::sub(tX, FLOOR_MAGIC), y0f = R::sub(tY, FLOOR_MAGIC);
            const float wx1 = (x0f + 1.f) - ix, wx0 = ix - x0f, wy1 = (y0f + 1.f) - iy, wy0 = iy - y0f;
            const float w_nw = wx1 * wy1, w_ne = wx0 * wy1, w_sw = wx1 * wy0, w_se = wx0 * wy0;
            float go[NC];
#pragma unroll
            for (int c = 0; c < NC; ++c) go[c] = j == 0 ? go2[c].x : go2[c].y;
            const uint32_t cell = ((unsigned)Y * (unsigned)BW + (unsigned)X) * 4u;
            // EDGE tiles only: taps in column / row -1 are outside the image
            const bool west_in = !EDGE || !(edge_x && ix < 0.f), north_in = !EDGE || !(edge_y && iy < 0.f);
            if (NEED_SRC && STRIDE1 && two_rounds) {
              // some neighbouring lanes share a cell (the map minifies here): first-of-cell lanes, then second-of-cell lanes
              const uint32_t a = cell + strip_base;
#pragma unroll
              for (int round = 0; round < 2; ++round) {
                const bool act = (round == 0) != same1;
                if (act && west_in && north_in) {
#pragma unroll
                  for (int c = 0; c < NC; ++c) tma::sts(a + c * SPLANE * 4, tma::lds(a + c * SPLANE * 4) + w_nw * go[c]);
                }
                __syncwarp();
                if (act && north_in) {
#pragma unroll
                  for (int c = 0; c < NC; ++c) tma::sts(a + (c * SPLANE + 1) * 4, tma::lds(a + (c * SPLANE + 1) * 4) + w_ne * go[c]);
                }
                __syncwarp();
                if (act && west_in) {
#pragma unroll
                  for (int c = 0; c < NC; ++c) tma::sts(a + (c * SPLANE + BW) * 4, tma::lds(a + (c * SPLANE + BW) * 4) + w_sw * go[c]);
                }
                __syncwarp();
                if (act) {
#pragma unroll
                  for (int c = 0; c < NC; ++c)
                    tma::sts(a + (c * SPLANE + BW + 1) * 4, tma::lds(a + (c * SPLANE + BW + 1) * 4) + w_se * go[c]);
                }
                __syncwarp();
              }
            } else if (NEED_SRC) {
              const uint32_t a = cell + strip_base;
              // tap by tap: lanes hit distinct cells inside one instruction; __syncwarp orders the taps
              if (west_in && north_in) {
#pragma unroll
                for (int c = 0; c < NC; ++c) tma::sts(a + c * SPLANE * 4, tma::lds(a + c * SPLANE * 4) + w_nw * go[c]);
              }
              __syncwarp();
              if (north_in) {
#pragma unroll
                for (int c = 0; c < NC; ++c) tma::sts(a + (c * SPLANE + 1) * 4, tma::lds(a + (c * SPLANE + 1) * 4) + w_ne * go[c]);
              }
              __syncwarp();
              if (west_in) {
#pragma unroll
                for (int c = 0; c < NC; ++c) tma::sts(a + (c * SPLANE + BW) * 4, tma::lds(a + (c * SPLANE + BW) * 4) + w_sw * go[c]);
              }
              __syncwarp();
#pragma unroll
              for (int c = 0; c < NC; ++c)
                tma::sts(a + (c * SPLANE + BW + 1) * 4, tma::lds(a + (c * SPLANE + BW + 1) * 4) + w_se * go[c]);
              __syncwarp();
            }
            if (NEED_M) {
              const uint32_t t = cell + win_base;
              // s_tap = sum_c gout[c] * src[c, tap]; then the two bilinear derivatives
              float s_nw = 0.f, s_ne = 0.f, s_sw = 0.f, s_se = 0.f;
#pragma unroll
              for (int c = 0; c < NC; ++c) {
                s_nw = fmaf(go[c], (west_in && north_in) ? tma::lds(t + (c * SPLANE) * 4) : 0.f, s_nw);
                s_ne = fmaf(go[c], north_in ? tma::lds(t + (c * SPLANE + 1) * 4) : 0.f, s_ne);
                s_sw = fmaf(go[c], west_in ? tma::lds(t + (c * SPLANE + BW) * 4) : 0.f, s_sw);
                s_se = fmaf(go[c], tma::lds(t + (c * SPLANE + BW + 1) * 4), s_se);
              }
              gix = (s_ne - s_nw) * wy1 + (s_se - s_sw) * wy0;
              giy = (s_sw - s_nw) * wx1 + (s_se - s_ne) * wx0;
            }
          } else if (live) {
            // exact per-pixel path (the unpadded coordinate is re-clamped inside for 'border')
            const float2 g = bwd_pixel_global<NC, PAD, NEED_SRC, NEED_M>(p, b, y, x, ix, iy);
            gix = g.x;
            giy = g.y;
          }
          if (NEED_M && live) {
            const float dgx = gix * ux_scale * px, dgy = giy * uy_scale * py;
            const float ax = dgx * rden, ay = dgy * rden;
            pm[0] += ax * bxv[j]; pm[1] += ax * byr; pm[2] += ax;
            pm[3] += ay * bxv[j]; pm[4] += ay * byr; pm[5] += ay;
            if (PROJ) {
              const float az = -(ax * gx + ay * gy);
              pm[6] += az * bxv[j]; pm[7] += az * byr; pm[8] += az;
            }
          }
        }
      }
      };
      if (edge_x || edge_y) rows(std::true_type{});  // warp-uniform
      else rows(std::false_type{});
      // flush the strip: one TMA reduce-add per warp and tile
      if (NEED_SRC) {
        tma::fence_proxy_async();
        __syncwarp();
        if (lane == 0 && sox < 0x10000000 && soy < 0x10000000) {
          tma::reduce_add_3d(&tmap_gsrc, strip_u32, sox, soy, b * NC);
          tma::bulk_commit();
        }
      }
      __syncwarp();
    }
    if (NEED_M) {
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        float v = pm[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        pm[k] = v;
      }
      if (lane == 0) {
        float* rec = p.records + ((size_t)record_row * TMA_CONSUMER_WARPS + slice) * 9;
#pragma unroll
        for (int k = 0; k < 9; ++k) rec[k] = pm[k];
        if (slice == 0) p.record_batch[record_row] = b;
      }
    }
  }
  if (NEED_SRC && lane == 0) tma::bulk_wait0();  // reductions done before exit
}

}  // namespace kb200
