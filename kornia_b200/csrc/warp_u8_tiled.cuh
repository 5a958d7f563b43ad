// kornia_b200 -- tiled uint8 ingest warp (fp32 out, bilinear, zeros / border / reflection / fill, C in {1,3,4}).
//
// warp_fwd_u8hwc (warp_u8.cuh) converts every tap where it is gathered: 4 taps x C conversions per output pixel, each
// behind its own byte load.  Here one CTA owns a 64 x 32 output tile, in the structure of remap_tiled_kernel
// (remap_tiled.cuh, hardware-verified):
//   1. every thread maps its 8 pixels (the reference's coordinate chain, IEEE divisions) and keeps the source
//      coordinates in registers;
//   2. the CTA reduces their bounding box (warp shuffles + one shared round) and thread 0 places a 72 x 40 pixel window;
//   3. all 256 threads stage the window in groups of 4 pixels: C aligned 32-bit loads of the interleaved bytes (W % 4 == 0
//      and a window start on a multiple of 4 pixels keep every group aligned and on one side of the image edge), each
//      byte converted ONCE with the tap conversion of warp_u8.cuh, one 16-byte store per channel into a planar fp32 box
//      in shared memory -- 1.4 x C conversions per output pixel instead of 4 x C -- out-of-image texels as zeros
//      (= 'zeros' padding);
//   4. pixels whose taps lie inside the window blend from shared memory with remap_tiled_kernel's arithmetic, the rest
//      take the exact per-pixel path of warp_fwd_u8hwc -- bit-identical to that kernel by construction.
// No TMA: the source is not a tensor the TMA unit could de-interleave AND convert; plain loads, shared stores and two
// __syncthreads, so the CPU-side emulator (tools/hostemu) models everything this kernel does except speed.
// Algorithmic bytes per RGB pixel: 3 read + 12 written.
//
// KB200_U8_SIMPLE=1 forces warp_fwd_u8hwc (tests compare the two bit for bit).
#pragma once
#include "remap_tiled.cuh"
#include "warp_u8.cuh"

namespace kb200 {

// One pixel entirely through global memory: the arithmetic of warp_fwd_u8hwc (PixelSampler on the byte image).  Out of
// line, like careful_pixel of the fp32 kernel: eight inlined copies would triple the kernel's code for a path that near-
// identity maps never take.
template <int NC, int PAD, bool ALIGN>
__device__ __noinline__ void u8_exact_pixel(const unsigned char* img, int H, int W, float ux, float uy, float scale, bool divide, float* o,
                                            size_t oplane, const float* fill) {
  PixelSampler<float, KB200_BILINEAR, PAD> S;
  S.prepare(ux, uy, H, W, ALIGN);
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const float v = S.sample_with([&](int off) { return value_of_byte(__ldg(img + (size_t)off * NC + c), scale, divide); });
    __stcs(o + c * oplane, S.finish(v, PAD == KB200_FILL ? ldg(fill + c) : 0.0f));
  }
}

#ifdef KB200_HOST_EMU
static long long u8t_fast_pixels = 0, u8t_exact_pixels = 0;  // tools/hostemu reports the share of the shared-memory path
#endif

// Coordinate source of the tile kernel: the affine / projective map of the warps (KIND_AFFINE, KIND_PROJ of
// warp_generic.cuh) or U8_KIND_LENS -- undistort_image (calibration/undistort.py:183-198) on decoder bytes: the lens model
// of remap_tiled.cuh:lens_distort evaluated per pixel, then remap's normalise -> unnormalise chain (align_corners=True),
// exactly as remap_tiled_kernel<NC, ZEROS, true, LENS=true> does on an fp32 image; output size = input size.
constexpr int U8_KIND_LENS = 3;

template <int NC, int PAD, int KIND, bool ALIGN>
__global__ void __launch_bounds__(256, KIND == U8_KIND_LENS ? 3 : 4) warp_u8_tiled_kernel(const __grid_constant__ WarpU8Params p) {
  using R = RN<float>;
  constexpr int TW = 64, TH = 32, BW = 72, BH = 40;
  constexpr int NJ = 2, RPW = 4;
  constexpr int PLANE = BW * BH;
  static_assert(BW % 4 == 0, "whole 4-pixel groups per window row");
  // reflection and fill: the window is clipped to pixels whose whole footprint is inside the image -- there the reflection
  // is the identity and the coverage of 'fill' (imgwarp.py:308-320: sample + (1 - sum of in-image weights) * fill) is complete
  constexpr bool INTERIOR = PAD == KB200_REFLECTION || PAD == KB200_FILL;
  constexpr bool PRECLAMP = PAD == KB200_BORDER;

  extern __shared__ __align__(128) unsigned char u8t_smem[];
  float* box = reinterpret_cast<float*>(u8t_smem);  // [NC][BH][BW]
  float* red = box + NC * PLANE;                    // [8 warps][4]
  float* win = red + 32;                            // lo_x, hi_x, lo_y, hi_y
  int* org = reinterpret_cast<int*>(win + 4);       // ox, oy, usable
  unsigned* kidx = reinterpret_cast<unsigned*>(org + 3);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tx = blockIdx.x, ty = blockIdx.y, b = blockIdx.z;
  const int H = p.H, W = p.W;
  const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1), Wf = (float)W, Hf = (float)H;
  const size_t oplane = (size_t)p.h * p.w;
  const int x0 = tx * TW + lane, y_base = ty * TH + warp * RPW;
  Mat3<float> m;
  float L[16];
  if (KIND == U8_KIND_LENS) {
#pragma unroll
    for (int k = 0; k < 16; ++k) L[k] = __ldg(p.lens + (size_t)b * 16 + k);
  } else {
    m.load(p.m + (p.Bm == 1 ? 0 : (size_t)b * 9));
  }
  // conversions.py:1487-1498 (remap's pixel -> [-1,1] step): factor = 2 / clamp(size - 1, eps)
  const float nfx = R::div(2.f, fmaxf(Wm1, 1e-8f)), nfy = R::div(2.f, fmaxf(Hm1, 1e-8f));
  const float scale = p.normalize == 1 ? RCP_255 : 1.0f;
  const bool divide = p.normalize == 2;
  float fillv[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) fillv[c] = PAD == KB200_FILL ? ldg(p.fill + c) : 0.0f;

  // ---- 1. coordinates of this thread's pixels
  float ux[RPW * NJ], uy[RPW * NJ];  // unnormalised, un-padded (what the exact path consumes)
  float lo_x = 3.0e38f, hi_x = -3.0e38f, lo_y = 3.0e38f, hi_y = -3.0e38f;
  bool finite = true;
  float bxv[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) bxv[j] = (KIND != U8_KIND_LENS && x0 + 32 * j < p.w) ? ldg(p.bx + x0 + 32 * j) : 0.f;
#pragma unroll
  for (int i = 0; i < RPW; ++i) {
    const int y = y_base + i;
    const float byv = (KIND != U8_KIND_LENS && y < p.h) ? ldg(p.by + y) : 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int x = x0 + 32 * j;
      const int u = i * NJ + j;
      float gx = 0.f, gy = 0.f, den;
      const bool live = x < p.w && y < p.h;
      if (live) {
        if (KIND == U8_KIND_LENS) {
          lens_distort(L, (float)x, (float)y, gx, gy);
          gx = R::sub(R::mul(nfx, gx), 1.f);
          gy = R::sub(R::mul(nfy, gy), 1.f);
        } else {
          map_point<float, KIND == KIND_PROJ>(m, bxv[j], byv, gx, gy, den);
        }
      }
      ux[u] = unnorm<ALIGN>(gx, Wm1, Wf);
      uy[u] = unnorm<ALIGN>(gy, Hm1, Hf);
      if (live) {
        float ix = ux[u], iy = uy[u];
        finite = finite && fabsf(ix) < 4.0e6f && fabsf(iy) < 4.0e6f;
        if (PRECLAMP) {
          ix = fminf(Wm1, fmaxf(ix, 0.f));
          iy = fminf(Hm1, fmaxf(iy, 0.f));
        }
        lo_x = fminf(lo_x, ix); hi_x = fmaxf(hi_x, ix);
        lo_y = fminf(lo_y, iy); hi_y = fmaxf(hi_y, iy);
      }
    }
  }
  // ---- 2. bounding box of the tile
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo_x = fminf(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o));
    hi_x = fmaxf(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
    lo_y = fminf(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o));
    hi_y = fmaxf(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, o));
  }
  finite = __all_sync(0xffffffffu, finite);
  if (lane == 0) {
    red[warp * 4 + 0] = finite ? lo_x : -3.0e38f;  // a non-finite coordinate anywhere disables the window
    red[warp * 4 + 1] = finite ? hi_x : 3.0e38f;
    red[warp * 4 + 2] = lo_y;
    red[warp * 4 + 3] = hi_y;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = red[0], bb = red[1], c = red[2], d = red[3];
    for (int wv = 1; wv < 8; ++wv) {
      a = fminf(a, red[wv * 4]); bb = fmaxf(bb, red[wv * 4 + 1]);
      c = fminf(c, red[wv * 4 + 2]); d = fmaxf(d, red[wv * 4 + 3]);
    }
    bool ok = a > -4.0e6f && bb < 4.0e6f && c > -4.0e6f && d < 4.0e6f && a <= bb && c <= d;
    const int x_lo = ok ? (int)floorf(a) : 0, x_hi = ok ? (int)floorf(bb) + 1 : 0;
    const int y_lo = ok ? (int)floorf(c) : 0, y_hi = ok ? (int)floorf(d) + 1 : 0;
    const int need_w = x_hi - x_lo + 1, need_h = y_hi - y_lo + 1;
    const int spare = BW - need_w - 3;
    const int ox = (x_lo - (spare > 0 ? spare / 2 : 0)) & ~3;  // window start on a multiple of 4 pixels: aligned words
    ok = ok && x_hi - ox + 1 <= BW && need_h <= BH;
    const int oy = ok ? y_lo - (BH - need_h) / 2 : 0;
    if (ok) {
      float wlx = (float)ox, whx = (float)(ox + BW - 1), wly = (float)oy, why = (float)(oy + BH - 1);
      if (INTERIOR) {
        wlx = fmaxf(wlx, 0.f); whx = fminf(whx, Wm1);
        wly = fmaxf(wly, 0.f); why = fminf(why, Hm1);
      }
      win[0] = wlx; win[1] = whx; win[2] = wly; win[3] = why;
      *kidx = (unsigned)(FLOOR_MAGIC_BITS + oy) * (unsigned)BW + (unsigned)(FLOOR_MAGIC_BITS + ox);
    } else {  // empty window: every pixel of the tile takes the exact path
      win[0] = win[2] = 1.f;
      win[1] = win[3] = 0.f;
      *kidx = 0;
    }
    org[0] = ok ? ox : 0; org[1] = oy; org[2] = ok ? 1 : 0;
  }
  __syncthreads();

  // ---- 3. stage the window: interleaved bytes -> planar fp32, every byte converted once.  Work item = 4 adjacent pixels
  // of a window row: NC aligned words in (4 * NC bytes; the window starts on a multiple of 4 pixels and W % 4 == 0, so a
  // group lies entirely inside or outside the image row), one 16-byte shared store per channel plane out.
  const unsigned char* img = p.src + (size_t)b * H * W * NC;
  if (org[2]) {
    const int ox = org[0], oy = org[1];
    constexpr int GROUPS = BW / 4;  // per window row
    for (int e = threadIdx.x; e < BH * GROUPS; e += 256) {
      const int r = e / GROUPS, g = e - r * GROUPS;
      const int gy = oy + r, gx = ox + 4 * g;
      uint32_t word[NC];
#pragma unroll
      for (int k = 0; k < NC; ++k) word[k] = 0;  // out-of-image texels are zeros ('zeros' padding; never blended otherwise)
      if ((unsigned)gy < (unsigned)H && (unsigned)gx < (unsigned)W) {
        const unsigned char* src = img + ((size_t)gy * W + gx) * NC;
#ifdef KB200_HOST_EMU
        if ((reinterpret_cast<uintptr_t>(src) & 3) != 0 || gx + 4 > W) emu::fail("misaligned or straddling 32-bit loads of the byte image");
#endif
#pragma unroll
        for (int k = 0; k < NC; ++k) word[k] = __ldg(reinterpret_cast<const uint32_t*>(src) + k);
      }
      float v[NC][4];
#pragma unroll
      for (int q = 0; q < 4 * NC; ++q)  // byte q of the group: pixel q / NC, channel q % NC (compile-time after unrolling)
        v[q % NC][q / NC] = value_of_level(level_of_word_byte(word[q / 4], q % 4), scale, divide);
#pragma unroll
      for (int c = 0; c < NC; ++c)
        *reinterpret_cast<float4*>(box + c * PLANE + r * BW + 4 * g) = make_float4(v[c][0], v[c][1], v[c][2], v[c][3]);
    }
  }
  __syncthreads();
  const float wlx = win[0], whx = win[1], wly = win[2], why = win[3];
  const uint32_t tbase = tma::smem_u32(box) - 4u * (*kidx);

  // ---- 4. sample
  float* obase = p.out + (size_t)b * NC * oplane;
#pragma unroll
  for (int i = 0; i < RPW; ++i) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int x = x0 + 32 * j, y = y_base + i;
      if (x >= p.w || y >= p.h) continue;
      const int u = i * NJ + j;
      float ix = ux[u], iy = uy[u];
      if (PRECLAMP) {
        ix = fminf(Wm1, fmaxf(ix, 0.f));
        iy = fminf(Hm1, fmaxf(iy, 0.f));
      }
      ix = interior_reflection<PAD, ALIGN>(ix);  // the window test and the taps below see the coordinate reflect_coord returns
      iy = interior_reflection<PAD, ALIGN>(iy);
      float* o = obase + (size_t)y * p.w + x;
#ifdef KB200_HOST_EMU
      ++((ix >= wlx && ix < whx && iy >= wly && iy < why) ? u8t_fast_pixels : u8t_exact_pixels);
#endif
      if (ix >= wlx && ix < whx && iy >= wly && iy < why) {
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
          if (PAD == KB200_FILL) {  // PixelSampler's coverage in tap order (all four taps in the image here), then finish()
            const float cover = R::add(R::add(R::add(R::add(0.f, w_nw), w_ne), w_sw), w_se);
            a = R::add(a, R::mul(R::sub(1.f, cover), fillv[c]));
          }
          __stcs(o + c * oplane, a);
        }
      } else {
        u8_exact_pixel<NC, PAD, ALIGN>(img, H, W, ux[u], uy[u], scale, divide, o, oplane, p.fill);
      }
    }
  }
}

static_assert(4 * 72 * 40 * 4 + 32 * 4 + 4 * 4 + 3 * 4 + 4 <= 48 * 1024, "the RGBA box fits the default dynamic shared-memory limit");
constexpr int U8T_SMEM_BYTES(int nc) { return nc * 72 * 40 * 4 + 32 * 4 + 4 * 4 + 3 * 4 + 4; }

}  // namespace kb200
