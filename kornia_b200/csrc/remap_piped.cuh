// kornia_b200 -- tiled remap forward, pipelined (fp32, bilinear, zeros/border/reflection, C in {1,3}; maps read from memory).
//
// Same per-pixel arithmetic as remap_tiled_kernel (remap_tiled.cuh: the normalise -> unnormalise chain of
// kornia/geometry/transform/imgwarp.py:688-702 + conversions.py:1487-1498 + GridSampler.h:27-35, taps from a TMA-staged
// 72 x 40 x C source box, everything else on the exact per-pixel path) -- bit-identical results -- with the dependent chain
// of that kernel taken off the critical path.
//
// remap_tiled_kernel stalls on long-scoreboard waits and on its mbarrier spin.  One CTA per tile there runs
//     map loads (DRAM latency) -> bounding box -> CTA barrier -> box load (DRAM latency again) -> blend -> exit
// and only the four co-resident CTAs of an SM overlap each other's waits: too few bytes in flight for HBM speed.
// Here persistent CTAs (8 consumer warps + 1 producer warp, two per SM) walk strips of tiles and every load is a TMA load
// issued tiles ahead of its use:
//   * the map tiles (64 x 32 of map_x and of map_y) of tile t+2 are in flight while
//   * the consumer warps, before they blend tile t, take the coordinates of tile t+1 out of its map tile (handing the buffer
//     back at once), keep them in registers and publish their share of its bounding box; the producer warp folds the eight
//     shares and issues the 72 x 40 x C source box of tile t+1, which lands while tile t is blended.
//     (First version, measured: the producer warp reducing the whole 2048-pixel box itself took 6 us per tile and the eight
//     consumer warps waited on it -- 1.22 ms against 0.88 ms for the one-CTA-per-tile kernel.)
// Shared memory: 2 x 34.6 KB boxes + 2 x 16 KB map tiles = 102 KB per CTA.  Algorithmic bytes: 8 (maps) + 12 + 12 per RGB pixel.
#pragma once
#include "remap_tiled.cuh"

namespace kb200 {

constexpr int REMAP_PIPED_STAGES = 2;

template <int NC, int PAD, bool ALIGN>
__global__ void __launch_bounds__(TMA_THREADS, 2) remap_piped_kernel(const __grid_constant__ CUtensorMap tmap_src,
                                                                     const __grid_constant__ CUtensorMap tmap_mx,
                                                                     const __grid_constant__ CUtensorMap tmap_my,
                                                                     const __grid_constant__ RemapTiledParams p) {
  using R = RN<float>;
  constexpr int TW = 64, TH = 32, BW = 72, BH = 40;
  constexpr int NJ = 2, RPW = 4, NS = REMAP_PIPED_STAGES, NU = RPW * NJ;
  constexpr int PLANE = BW * BH;
  constexpr int BOX_FLOATS = NC * PLANE, MAP_FLOATS = TW * TH;
  constexpr uint32_t BOX_BYTES = BOX_FLOATS * 4, MAP_BYTES = MAP_FLOATS * 4;
  // 'reflection': the fast path reflects the coordinate itself (reflect_clip_near, sampler.cuh: bit-identical to reflect_coord +
  // clip_coord), so border tiles stay in shared memory -- the one-CTA-per-tile kernel restricts its fast path to interior pixels
  constexpr bool REFLECT = PAD == KB200_REFLECTION;
  constexpr bool PRECLAMP = PAD == KB200_BORDER;
  static_assert(TH == TMA_CONSUMER_WARPS * RPW && TW == 32 * NJ, "thread mapping");

  extern __shared__ __align__(128) unsigned char remap_piped_smem[];
  float* boxes = reinterpret_cast<float*>(remap_piped_smem);                 // [NS][NC][BH][BW]
  float* maps = boxes + NS * BOX_FLOATS;                                     // [NS][2][TH][TW]: map_x tile, then map_y tile
  float* red = maps + NS * 2 * MAP_FLOATS;                                   // [NS][8 warps][4]: per-warp bounding boxes
  uint64_t* box_full = reinterpret_cast<uint64_t*>(red + NS * TMA_CONSUMER_WARPS * 4);
  uint64_t* box_empty = box_full + NS;
  uint64_t* map_full = box_empty + NS;
  uint64_t* map_empty = map_full + NS;
  uint64_t* red_full = map_empty + NS;
  StageInfo* info = reinterpret_cast<StageInfo*>(red_full + NS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < NS; ++i) {
      tma::mbar_init(&box_full[i], 1);
      tma::mbar_init(&box_empty[i], TMA_CONSUMER_WARPS);
      tma::mbar_init(&map_full[i], 1);
      tma::mbar_init(&map_empty[i], TMA_CONSUMER_WARPS);
      tma::mbar_init(&red_full[i], TMA_CONSUMER_WARPS);
    }
    tma::fence_barrier_init();
  }
  __syncthreads();

  const int tiles_x = ceil_div(p.w, TW), tiles_y = ceil_div(p.h, TH);
  const Segments segs(p.B * tiles_y, tiles_x);
  const int H = p.H, W = p.W;
  const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1), Wf = (float)W, Hf = (float)H;
  // conversions.py:1487-1498: factor = 2 / clamp(size - 1, eps)
  const float fx = R::div(2.f, fmaxf(Wm1, 1e-8f)), fy = R::div(2.f, fmaxf(Hm1, 1e-8f));
  const bool normalized = p.normalized != 0;

  // A walk of this CTA's tile sequence; n = index of the current tile in it.
  struct Walk {
    int seg, strip, tx0, tx1, cursor, tx, n;
    bool live;
  };
  auto walk_next = [&](Walk& wk) {
    if (wk.live && wk.tx + 1 < wk.tx1) {
      ++wk.tx;
      ++wk.n;
      return;
    }
    const bool first = wk.seg == 0;
    wk.live = segs.get(wk.seg, wk.strip, wk.tx0, wk.tx1, wk.cursor);
    ++wk.seg;
    wk.tx = wk.tx0;
    if (!first) ++wk.n;
  };

  if (warp == TMA_CONSUMER_WARPS) {
    // ------------------------------------------------------------------ producer warp: issues every load
    if (tma::elect_one()) {
      tma::prefetch_map(&tmap_src);
      tma::prefetch_map(&tmap_mx);
      tma::prefetch_map(&tmap_my);
    }
    Walk mw{0, 0, 0, 0, 0, 0, 0, false}, xw = mw;
    auto map_issue = [&]() {  // all lanes; loads the map tiles of mw's tile, then steps
      if (!mw.live) return;
      const int s = mw.n % NS;
      tma::mbar_wait(&map_empty[s], ((mw.n / NS) & 1) ^ 1);
      if (tma::elect_one()) {
        const int b = mw.strip / tiles_y, ty = mw.strip - b * tiles_y;
        const int bm = p.Bmap == 1 ? 0 : b;
        float* dst = maps + s * 2 * MAP_FLOATS;
        tma::mbar_arrive_expect_tx(&map_full[s], 2 * MAP_BYTES);
        tma::load_3d(dst, &tmap_mx, &map_full[s], mw.tx * TW, ty * TH, bm);
        tma::load_3d(dst + MAP_FLOATS, &tmap_my, &map_full[s], mw.tx * TW, ty * TH, bm);
      }
      __syncwarp();
      walk_next(mw);
    };
    walk_next(mw);
    walk_next(xw);
    map_issue();
    map_issue();
    while (xw.live) {
      const int s = xw.n % NS;
      const uint32_t phase = (xw.n / NS) & 1;
      const int b = xw.strip / tiles_y;
      // the consumers reduced the bounding box of this tile to one entry per warp while they blended the tile before it
      tma::mbar_wait(&red_full[s], phase);
      const float* rd = red + (s * TMA_CONSUMER_WARPS + (lane & 7)) * 4;
      float lo_x = rd[0], hi_x = rd[1], lo_y = rd[2], hi_y = rd[3];
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        lo_x = fminf(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o));
        hi_x = fmaxf(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
        lo_y = fminf(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o));
        hi_y = fmaxf(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, o));
      }
      tma::mbar_wait(&box_empty[s], phase ^ 1);
      if (tma::elect_one()) {
        bool ok = lo_x > -4.0e6f && hi_x < 4.0e6f && lo_y > -4.0e6f && hi_y < 4.0e6f && lo_x <= hi_x && lo_y <= hi_y;
        const int x_lo = ok ? (int)floorf(lo_x) : 0, x_hi = ok ? (int)floorf(hi_x) + 1 : 0;
        const int y_lo = ok ? (int)floorf(lo_y) : 0, y_hi = ok ? (int)floorf(hi_y) + 1 : 0;
        const int need_w = x_hi - x_lo + 1, need_h = y_hi - y_lo + 1;
        const int spare = BW - need_w - 3;
        const int ox = (x_lo - (spare > 0 ? spare / 2 : 0)) & ~3;  // TMA: 16-byte aligned box start
        ok = ok && x_hi - ox + 1 <= BW && need_h <= BH;
        StageInfo si;
        si.inner = 0;
        if (ok) {
          const int oy = y_lo - (BH - need_h) / 2;
          si.lo_x = (float)ox; si.hi_x = (float)(ox + BW - 1);
          si.lo_y = (float)oy; si.hi_y = (float)(oy + BH - 1);
          si.k = (unsigned)(FLOOR_MAGIC_BITS + oy) * (unsigned)BW + (unsigned)(FLOOR_MAGIC_BITS + ox);
          info[s] = si;
          tma::mbar_arrive_expect_tx(&box_full[s], BOX_BYTES);
          tma::load_3d(boxes + s * BOX_FLOATS, &tmap_src, &box_full[s], ox, oy, b * NC);
        } else {
          si.lo_x = si.lo_y = 1.f;  // empty interval: nothing is served from the box
          si.hi_x = si.hi_y = 0.f;
          si.k = 0;
          info[s] = si;
          tma::mbar_arrive(&box_full[s]);
        }
      }
      __syncwarp();
      walk_next(xw);
      map_issue();  // two tiles ahead of the box just issued; its buffer came back when the consumers read that tile's maps
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warps
  const size_t oplane = (size_t)p.h * p.w, splane = (size_t)H * W;
  // Coordinates of this thread's eight pixels of walk wk's tile, out of its map tile (which goes back to the producer at once),
  // and this warp's share of the tile's bounding box, published for the producer.
  auto stage_coordinates = [&](const Walk& wk, float (&ux)[NU], float (&uy)[NU], unsigned& farmask) {
    farmask = 0u;
    const int s = wk.n % NS;
    const int ty = wk.strip % tiles_y;
    const int x0 = wk.tx * TW + lane, y_base = ty * TH + warp * RPW;
    tma::mbar_wait(&map_full[s], (wk.n / NS) & 1);
    const float* mxs = maps + s * 2 * MAP_FLOATS + (warp * RPW) * TW + lane;
    const float* mys = mxs + MAP_FLOATS;
    float gx[NU], gy[NU];
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      gx[u] = mxs[(u / NJ) * TW + 32 * (u % NJ)];
      gy[u] = mys[(u / NJ) * TW + 32 * (u % NJ)];
    }
    __syncwarp();
    if (lane == 0) tma::mbar_arrive(&map_empty[s]);
    float lo_x = 3.0e38f, hi_x = -3.0e38f, lo_y = 3.0e38f, hi_y = -3.0e38f;
    bool finite = true;
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      float a = gx[u], c = gy[u];
      if (!normalized) {
        a = R::sub(R::mul(fx, a), 1.f);
        c = R::sub(R::mul(fy, c), 1.f);
      }
      ux[u] = unnorm<ALIGN>(a, Wm1, Wf);
      uy[u] = unnorm<ALIGN>(c, Hm1, Hf);
      if (x0 + 32 * (u % NJ) < p.w && y_base + u / NJ < p.h) {  // pixels beyond the output read the TMA zero fill and are skipped
        float ix = ux[u], iy = uy[u];
        finite = finite && fabsf(ix) < 4.0e6f && fabsf(iy) < 4.0e6f;
        if (PRECLAMP) {
          ix = fminf(Wm1, fmaxf(ix, 0.f));
          iy = fminf(Hm1, fmaxf(iy, 0.f));
        }
        bool far = false;  // 'reflection', more than one span outside the image: exact path, not part of the box
        if (REFLECT) {
          ix = reflect_clip_near<ALIGN>(ix, W, far);
          iy = reflect_clip_near<ALIGN>(iy, H, far);
        }
        if (!far) {
          lo_x = fminf(lo_x, ix); hi_x = fmaxf(hi_x, ix);
          lo_y = fminf(lo_y, iy); hi_y = fmaxf(hi_y, iy);
        } else {
          farmask |= 1u << u;
        }
        // The PADDED coordinate is what stays in registers: the clamp is idempotent, and so is the near reflection (its half-pixel
        // round trip returns the value it produced: tools/hostemu test_reflect_near), so the exact path may pad it again.  Only a
        // `far` pixel needs its raw coordinate, and reads its map entry again for it.
        ux[u] = ix;
        uy[u] = iy;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo_x = fminf(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o));
      hi_x = fmaxf(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
      lo_y = fminf(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o));
      hi_y = fmaxf(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, o));
    }
    finite = __all_sync(0xffffffffu, finite);
    if (lane == 0) {
      float* rd = red + (s * TMA_CONSUMER_WARPS + warp) * 4;
      rd[0] = finite ? lo_x : -3.0e38f;  // a non-finite coordinate anywhere disables the box
      rd[1] = finite ? hi_x : 3.0e38f;
      rd[2] = lo_y;
      rd[3] = hi_y;
      tma::mbar_arrive(&red_full[s]);
    }
  };

  Walk cw{0, 0, 0, 0, 0, 0, 0, false}, nw = cw;
  walk_next(cw);
  walk_next(nw);
  walk_next(nw);  // one tile ahead
  float ux[NU], uy[NU];
  unsigned farmask = 0u;
  if (cw.live) stage_coordinates(cw, ux, uy, farmask);
  while (cw.live) {
    const int s = cw.n % NS;
    const int b = cw.strip / tiles_y, ty = cw.strip - b * tiles_y;
    const int x0 = cw.tx * TW + lane, y_base = ty * TH + warp * RPW;
    // ---- 1. the next tile's coordinates and bounding box: the producer turns them into a box load while this tile is blended
    float nux[NU], nuy[NU];
    unsigned nfarmask = 0u;
    if (nw.live) stage_coordinates(nw, nux, nuy, nfarmask);
    // ---- 2. this tile's box
    tma::mbar_wait(&box_full[s], (cw.n / NS) & 1);
    const StageInfo si = info[s];
    const uint32_t tbase = tma::smem_u32(boxes + s * BOX_FLOATS) - 4u * si.k;
    const float* sp = p.src + (size_t)b * NC * splane;
    float* obase = p.out + (size_t)b * NC * oplane;
    // ---- 3. sample
#pragma unroll
    for (int i = 0; i < RPW; ++i) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int x = x0 + 32 * j, y = y_base + i;
        if (x >= p.w || y >= p.h) continue;
        const int u = i * NJ + j;
        const float ix = ux[u], iy = uy[u];  // padded already (stage_coordinates)
        const bool far = REFLECT && ((farmask >> u) & 1u) != 0u;
        float* o = obase + (size_t)y * p.w + x;
        if (!far && ix >= si.lo_x && ix < si.hi_x && iy >= si.lo_y && iy < si.hi_y) {
          const float tX = __fadd_rd(ix, FLOOR_MAGIC), tY = __fadd_rd(iy, FLOOR_MAGIC);
          const uint32_t a0 = ((unsigned)__float_as_int(tY) * (unsigned)BW + (unsigned)__float_as_int(tX)) * 4u + tbase;
          const float x0f = R::sub(tX, FLOOR_MAGIC), y0f = R::sub(tY, FLOOR_MAGIC);
          const float wx1 = R::sub(R::add(x0f, 1.f), ix), wx0 = R::sub(ix, x0f);
          const float wy1 = R::sub(R::add(y0f, 1.f), iy), wy0 = R::sub(iy, y0f);
          const float w_nw = R::mul(wx1, wy1), w_ne = R::mul(wx0, wy1), w_sw = R::mul(wx1, wy0), w_se = R::mul(wx0, wy0);
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            float a = R::fma(tma::lds(a0 + (c * PLANE) * 4), w_nw, 0.f);
            a = R::fma(tma::lds(a0 + (c * PLANE + 1) * 4), w_ne, a);
            a = R::fma(tma::lds(a0 + (c * PLANE + BW) * 4), w_sw, a);
            a = R::fma(tma::lds(a0 + (c * PLANE + BW + 1) * 4), w_se, a);
            __stcs(o + c * oplane, a);
          }
        } else {
          float ex = ix, ey = iy;
          if (far) {  // beyond two spans: the raw coordinate, from the map entry (an L2 hit)
            const size_t at = (p.Bmap == 1 ? 0 : (size_t)b * oplane) + (size_t)y * p.w + x;
            float a = __ldg(p.map_x + at), c = __ldg(p.map_y + at);
            if (!normalized) {
              a = R::sub(R::mul(fx, a), 1.f);
              c = R::sub(R::mul(fy, c), 1.f);
            }
            ex = unnorm<ALIGN>(a, Wm1, Wf);
            ey = unnorm<ALIGN>(c, Hm1, Hf);
          }
          PixelSampler<float, KB200_BILINEAR, PAD> S;
          S.prepare(ex, ey, H, W, ALIGN);
#pragma unroll
          for (int c = 0; c < NC; ++c) __stcs(o + c * oplane, S.sample(sp + c * splane));
        }
      }
    }
    __syncwarp();
    if (lane == 0) tma::mbar_arrive(&box_empty[s]);
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      ux[u] = nux[u];
      uy[u] = nuy[u];
    }
    farmask = nfarmask;
    walk_next(cw);
    walk_next(nw);
  }
}

// KB200_EUNSUPPORTED (maps not TMA-addressable, switch off) -> remap_tiled_forward's own kernel.
int remap_piped_forward(const float* src, const float* map_x, const float* map_y, float* out, int B, int C, int H, int W, int h, int w,
                        int Bmap, int normalized, int pad, int align, cudaStream_t st);

}  // namespace kb200
