// Executes the kernel templates of kornia_b200/csrc on the CPU (hostemu.h) and compares them BIT FOR BIT with scalar
// restatements of the same arithmetic.  Covers the pipelined kernels and, as a check of the emulator itself, the
// kernels they derive from.
//
//   make -C tools/hostemu && tools/hostemu/run_emu          (or: python tools/hostemu/run.py)
//
// x86 fmaf() is correctly rounded and the build uses -ffp-contract=off, so fp32 results are those of the device
// intrinsics (__fmaf_rn, __fmul_rn, ...).  What this does NOT cover: timing, occupancy, bank conflicts, the real TMA
// unit and the memory model of the async proxy -- a pass here means "the index arithmetic, the pipeline bookkeeping and
// the barriers are consistent", not "runs on the GPU".
#include "hostemu.h"

#include "../../kornia_b200/csrc/filter2d_tiled.cuh"
#include "../../kornia_b200/csrc/gradient_tiled.cuh"
#include "../../kornia_b200/csrc/ssim_vwalk.cuh"
#include "../../kornia_b200/csrc/remap_tiled.cuh"
#include "ref_ssim_tiled.cuh"
#include "../../kornia_b200/csrc/warp_bwd_tma2.cuh"
#include "../../kornia_b200/csrc/warp_u8_tiled.cuh"

#include <random>
#include <string>

namespace kb200 {
alignas(128) unsigned char sept_smem[256 * 1024];
alignas(128) unsigned char f2d_smem[256 * 1024];
alignas(128) unsigned char gradt_smem[256 * 1024];
alignas(128) unsigned char ssimv_smem[256 * 1024];
alignas(128) float ssim_smem[64 * 1024];
alignas(128) unsigned char remap_smem[256 * 1024];
alignas(128) unsigned char tma_smem[256 * 1024];
alignas(128) unsigned char bwd2_smem[256 * 1024];
alignas(128) unsigned char u8t_smem[256 * 1024];
void set_error(const char*, ...) {}
}  // namespace kb200

using namespace kb200;

static std::mt19937 rng(1234);
static std::vector<float> randv(size_t n, float lo = 0.f, float hi = 1.f) {
  std::uniform_real_distribution<float> d(lo, hi);
  std::vector<float> v(n);
  for (auto& x : v) x = d(rng);
  return v;
}
static float* aligned(std::vector<float>& store, size_t n) {  // 128-byte aligned view into a vector
  store.assign(n + 64, -777.f);
  return reinterpret_cast<float*>(((size_t)store.data() + 127) & ~(size_t)127);
}
static int fold(int q, int n, int border) {
  if (q >= 0 && q < n) return q;
  if (border == KB200_CONSTANT) return -1;
  if (border == KB200_REPLICATE) return q < 0 ? 0 : n - 1;
  return q < 0 ? -q : 2 * (n - 1) - q;
}
static int failures = 0;
static void compare(const std::string& what, const float* got, const float* want, size_t n) {
  size_t bad = 0, first = 0;
  for (size_t i = 0; i < n; ++i)
    if (memcmp(got + i, want + i, 4) != 0 && !(got[i] == 0.f && want[i] == 0.f)) {
      if (!bad) first = i;
      ++bad;
    }
  if (bad) {
    printf("FAIL %-72s %zu / %zu differ, first at %zu: got %.9g want %.9g\n", what.c_str(), bad, n, first, got[first], want[first]);
    ++failures;
  } else {
    printf("ok   %s\n", what.c_str());
  }
}

// ------------------------------------------------------------------------------------------ separable filter
static void ref_sepfilter(const float* x, const float* kx, const float* ky, float* out, int planes, int C, int H, int W, int Bk, int K, int border) {
  const int h = (K - 1) / 2;
  std::vector<float> mid((size_t)H * W);
  for (int p = 0; p < planes; ++p) {
    const float* xp = x + (size_t)p * H * W;
    const float* kxp = kx + (size_t)((p / C) % Bk) * K;
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        float a = 0.f;
        for (int j = 0; j < K; ++j) {
          const int sx = fold(xx + j - h, W, border);
          a = fmaf(kxp[j], sx < 0 ? 0.f : xp[(size_t)y * W + sx], a);
        }
        mid[(size_t)y * W + xx] = a;
      }
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        float a = 0.f;
        for (int i = 0; i < K; ++i) {
          const int sy = fold(y + i - h, H, border);
          a = fmaf(ky[i], sy < 0 ? 0.f : mid[(size_t)sy * W + xx], a);
        }
        out[(size_t)p * H * W + (size_t)y * W + xx] = a;
      }
  }
}

template <int K, int BORDER>
static void test_sepfilter(int B, int C, int H, int W, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  const int planes = B * C;
  std::vector<float> xs, o1s, o2s;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  auto kx = randv((size_t)B * K, -1.f, 1.f), ky = randv(K, -1.f, 1.f);
  std::vector<float> want((size_t)planes * H * W);
  ref_sepfilter(x, kx.data(), ky.data(), want.data(), planes, C, H, W, B, K, BORDER);
  float* o1 = aligned(o1s, want.size());
  float* o2 = aligned(o2s, want.size());
  const std::string tag = "K=" + std::to_string(K) + " border=" + std::to_string(BORDER) + " " + std::to_string(B) + "x" + std::to_string(C) + "x" +
                          std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
  {  // the hardware-verified strip-walking kernel: checks the emulator
    const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
    SepTiledParams p{kx.data(), ky.data(), o1, C, H, W, B, 1, planes, x, 0.f};
    emu::launch(grid, dim3(256), [&] { sepfilter_tiled_kernel<K, BORDER, false>(map, p); });
    compare("sepfilter_tiled_kernel (verified on hw) " + tag, o1, want.data(), want.size());
  }
  if (K <= 11) {  // unsharp_mask epilogue against the plain filter blended on the host (|w| < 0.5 and >= 0.5 take different forms)
    const float wts[2] = {0.3f, 2.0f};
    const float wt = wts[(H + W) & 1];
    std::vector<float> blended(want.size());
    for (size_t i = 0; i < want.size(); ++i) blended[i] = lerp_like_torch(o1[i], x[i], wt);
    const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
    SepTiledParams p{kx.data(), ky.data(), o2, C, H, W, B, 1, planes, x, wt};
    emu::launch(grid, dim3(256), [&] { sepfilter_tiled_kernel<K, BORDER, true>(map, p); });
    compare("sepfilter_tiled_kernel<LERP> vs lerp of the plain filter " + tag, o2, blended.data(), want.size());
  }
}

// ------------------------------------------------------------------------------------------ filter2d / pyrdown / derivatives
static void ref_filter2d(const float* x, const float* k, int nout, float* out, int planes, int H, int W, int K, int border) {
  const int h = (K - 1) / 2;
  for (int p = 0; p < planes; ++p)
    for (int o = 0; o < nout; ++o)
      for (int y = 0; y < H; ++y)
        for (int xx = 0; xx < W; ++xx) {
          float a = 0.f;
          for (int i = 0; i < K; ++i)
            for (int j = 0; j < K; ++j) {
              const int sy = fold(y + i - h, H, border), sx = fold(xx + j - h, W, border);
              a = fmaf(k[(o * K + i) * K + j], (sy < 0 || sx < 0) ? 0.f : x[(size_t)p * H * W + (size_t)sy * W + sx], a);
            }
          out[(((size_t)p * nout + o) * H + y) * W + xx] = a;
        }
}

template <int BORDER>
static void test_pyrdown(int planes, int H, int W, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  std::vector<float> xs, os, fs;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  float taps[25];
  const float b5[5] = {1, 4, 6, 4, 1};
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 5; ++j) taps[i * 5 + j] = b5[i] * b5[j] / 256.f;
  std::vector<float> full((size_t)planes * H * W), want((size_t)planes * (H / 2) * (W / 2));
  ref_filter2d(x, taps, 1, full.data(), planes, H, W, 5, BORDER);
  for (int p = 0; p < planes; ++p)
    for (int y = 0; y < H / 2; ++y)
      for (int xx = 0; xx < W / 2; ++xx) {
        const float* f = full.data() + (size_t)p * H * W + (size_t)(2 * y) * W + 2 * xx;
        want[((size_t)p * (H / 2) + y) * (W / 2) + xx] = 0.25f * ((f[0] + f[1]) + (f[W] + f[W + 1]));
      }
  const std::string tag = "border=" + std::to_string(BORDER) + " " + std::to_string(planes) + "x" + std::to_string(H) + "x" + std::to_string(W) +
                          " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
  const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + 4, 1);
  {
    float* o = aligned(fs, full.size());
    F2dTiledParams p{taps, o, 1, H, W, 1, planes};
    emu::launch(grid, dim3(256), [&] { filter2d_tiled_kernel<5, BORDER, false>(map, p); });
    compare("filter2d_tiled_kernel<5> (verified on hw) " + tag, o, full.data(), full.size());
  }
  {
    float* o = aligned(os, want.size());
    F2dTiledParams p{taps, o, 1, H, W, 1, planes};
    emu::launch(grid, dim3(256), [&] { filter2d_tiled_kernel<5, BORDER, true>(map, p); });
    compare("filter2d_tiled_kernel<5, DOWN2> (pyrdown)  " + tag, o, want.data(), want.size());
  }
}

template <int K, int BORDER>
static void test_filter2d(int planes, int H, int W, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  std::vector<float> xs, os;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  auto taps = randv(K * K, -1.f, 1.f);
  std::vector<float> want((size_t)planes * H * W);
  ref_filter2d(x, taps.data(), 1, want.data(), planes, H, W, K, BORDER);
  float* o = aligned(os, want.size());
  const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
  F2dTiledParams p{taps.data(), o, 1, H, W, 1, planes};
  emu::launch(grid, dim3(256), [&] { filter2d_tiled_kernel<K, BORDER, false>(map, p); });
  compare("filter2d_tiled_kernel (verified on hw) K=" + std::to_string(K) + " border=" + std::to_string(BORDER) + " " + std::to_string(planes) + "x" +
              std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"),
          o, want.data(), want.size());
}

template <int K, int NOUT, bool MAG>
static void test_gradient(int planes, int H, int W, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  std::vector<float> xs, os;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  GradTiledParams p;
  p.H = H; p.W = W; p.planes = planes; p.eps = 1e-6f;
  auto t = randv(NOUT * K * K, -1.f, 1.f);
  for (int e = 0; e < NOUT * K * K; ++e) p.taps[e] = (e % 4 == 1) ? 0.f : t[e];  // some exact zeros, like the Sobel stencils
  std::vector<float> d((size_t)planes * NOUT * H * W), want;
  ref_filter2d(x, p.taps, NOUT, d.data(), planes, H, W, K, KB200_REPLICATE);
  if (MAG) {
    want.resize((size_t)planes * H * W);
    for (int pl = 0; pl < planes; ++pl)
      for (size_t i = 0; i < (size_t)H * W; ++i) {
        const float gx = d[((size_t)pl * 2) * H * W + i], gy = d[((size_t)pl * 2 + 1) * H * W + i];
        want[(size_t)pl * H * W + i] = sqrtf((gx * gx + gy * gy) + p.eps);
      }
  } else {
    want = d;
  }
  p.out = aligned(os, want.size());
  const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
  emu::launch(grid, dim3(256), [&] { grad_tiled_kernel<K, NOUT, MAG>(map, p); });
  compare("grad_tiled_kernel K=" + std::to_string(K) + " NOUT=" + std::to_string(NOUT) + (MAG ? " MAG " : "     ") + std::to_string(planes) + "x" +
              std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"),
          p.out, want.data(), want.size());
}

// ------------------------------------------------------------------------------------------ SSIM
template <int K>
static void test_ssim(int planes, int H, int W, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  std::vector<float> as, bs, o1s, o2s;
  const size_t n = (size_t)planes * H * W;
  float* a = aligned(as, n);
  float* b = aligned(bs, n);
  for (size_t i = 0; i < n; ++i) {
    a[i] = randv(1)[0];
    b[i] = std::min(1.f, std::max(0.f, a[i] + randv(1, -0.1f, 0.1f)[0]));
  }
  auto taps = randv(K, 0.f, 1.f);
  const float C1 = 1e-4f, C2 = 9e-4f, eps = 1e-12f;
  const std::string tag = "K=" + std::to_string(K) + " " + std::to_string(planes) + "x" + std::to_string(H) + "x" + std::to_string(W) +
                          " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
  float* o1 = aligned(o1s, n);
  {  // the hardware-verified gather kernel is the reference here
    SsimParams p;
    p.a = a; p.b = b; p.taps = taps.data(); p.out = o1; p.planes = planes; p.H = H; p.W = W;
    p.tiles_x = ceil_div(W, SSIM_TW); p.tiles_y = ceil_div(H, SSIM_TH); p.pair_ok = (W % 2 == 0); p.C1 = C1; p.C2 = C2; p.eps = eps;
    emu::launch((unsigned)(p.tiles_x * p.tiles_y * planes), dim3(256), [&] { ssim_tiled_kernel<K>(p); });
  }
  float* o2 = aligned(o2s, n);
  {
    const CUtensorMap ma = emu::make_map(a, W, H, planes, SSIMV_BW, SSIMV_TH, 1), mb = emu::make_map(b, W, H, planes, SSIMV_BW, SSIMV_TH, 1);
    const CUtensorMap pa = emu::make_map(a, W, H, planes, SSIMV_BW, K - 1, 1), pb = emu::make_map(b, W, H, planes, SSIMV_BW, K - 1, 1);
    SsimVParams p{taps.data(), o2, planes, H, W, C1, C2, eps};
    emu::launch(grid, dim3(256), [&] { ssim_vwalk_kernel<K>(ma, mb, pa, pb, p); });
  }
  compare("ssim_vwalk_kernel vs ssim_tiled_kernel " + tag, o2, o1, n);
}


// ------------------------------------------------------------------------------------------ remap / fused undistort
static float ref_remap_pixel(const float* plane, int H, int W, float mx, float my) {
  // conversions.py:1487-1498 (normalise), GridSampler.h:27-35 (unnormalise, align_corners=True), bilinear + zeros
  const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1);
  const float fx = 2.f / fmaxf(Wm1, 1e-8f), fy = 2.f / fmaxf(Hm1, 1e-8f);
  const float gx = fx * mx - 1.f, gy = fy * my - 1.f;
  const float ix = ((gx + 1.f) * 0.5f) * Wm1, iy = ((gy + 1.f) * 0.5f) * Hm1;
  if (!(fabsf(ix) < 4.0e6f && fabsf(iy) < 4.0e6f)) return 0.f;
  const float x0f = floorf(ix), y0f = floorf(iy);
  const float wx1 = (x0f + 1.f) - ix, wx0 = ix - x0f, wy1 = (y0f + 1.f) - iy, wy0 = iy - y0f;
  const int x0 = (int)x0f, y0 = (int)y0f;
  auto tap = [&](int y, int x) { return (y >= 0 && y < H && x >= 0 && x < W) ? plane[(size_t)y * W + x] : 0.f; };
  float a = fmaf(tap(y0, x0), wx1 * wy1, 0.f);
  a = fmaf(tap(y0, x0 + 1), wx0 * wy1, a);
  a = fmaf(tap(y0 + 1, x0), wx1 * wy0, a);
  a = fmaf(tap(y0 + 1, x0 + 1), wx0 * wy0, a);
  return a;
}

static void test_undistort(int B, int H, int W, bool lazy, bool strong = false) {
  emu::lazy_tma = lazy;
  emu::set_smem(remap_smem, sizeof(remap_smem));
  constexpr int C = 3;
  std::vector<float> ss, o1s, o2s, mxs, mys;
  const size_t n = (size_t)B * C * H * W, npix = (size_t)B * H * W;
  float* src = aligned(ss, n);
  for (size_t i = 0; i < n; ++i) src[i] = randv(1)[0];
  std::vector<float> lens((size_t)B * 16);
  for (int b = 0; b < B; ++b) {
    // strong: a fish-eye-like model whose maps leave the 8-row windows (and partly the image): the exact per-pixel path
    const float L[16] = {(strong ? 0.35f : 0.8f) * W + 3 * b, (strong ? 0.3f : 0.75f) * W, 0.5f * W - 3.f, 0.5f * H + 2.f, strong ? -0.45f : -0.21f, 0.07f, 0.002f, -0.003f, 0.01f, 0.04f, -0.02f, 0.004f, 0.003f, -0.001f, 0.002f, 0.0015f};
    memcpy(&lens[(size_t)b * 16], L, sizeof(L));
  }
  // the maps the host composition would hand to remap: lens_distort on the exact integer grid (the same device function)
  float* mx = aligned(mxs, npix);
  float* my = aligned(mys, npix);
  std::vector<float> want(n);
  for (int b = 0; b < B; ++b) {
    float L[16];
    memcpy(L, &lens[(size_t)b * 16], sizeof(L));
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        float a, c;
        lens_distort(L, (float)x, (float)y, a, c);
        mx[((size_t)b * H + y) * W + x] = a;
        my[((size_t)b * H + y) * W + x] = c;
        for (int ch = 0; ch < C; ++ch)
          want[(((size_t)b * C + ch) * H + y) * W + x] = ref_remap_pixel(src + ((size_t)b * C + ch) * H * W, H, W, a, c);
      }
  }
  const CUtensorMap map = emu::make_map(src, W, H, B * C, 72, 40, C);
  const dim3 grid(ceil_div(W, 64), ceil_div(H, 32), B);
  const std::string tag = std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) + (lazy ? " lazy" : " eager") + (strong ? " strong" : "");
  float* o1 = aligned(o1s, n);
  {
    RemapTiledParams p{src, mx, my, o1, B, H, W, H, W, B, 0, nullptr};
    emu::launch3(grid, dim3(256), [&] { remap_tiled_kernel<3, KB200_ZEROS, true, false>(map, p); });
    compare("remap_tiled_kernel (verified on hw) vs scalar bilinear " + tag, o1, want.data(), n);
  }
  float* o2 = aligned(o2s, n);
  {
    RemapTiledParams p{src, nullptr, nullptr, o2, B, H, W, H, W, B, 0, lens.data()};
    emu::launch3(grid, dim3(256), [&] { remap_tiled_kernel<3, KB200_ZEROS, true, true>(map, p); });
    compare("remap_tiled_kernel<LENS> (fused undistort) vs maps + remap " + tag, o2, o1, n);
  }
}


// ------------------------------------------------------------------------------------------ tiled warp forward (the headline kernel)
// the source as (W, H, planes), one map per box height of warp_fwd_tma (boxes of one plane, BW wide)
template <int BW, int BH>
static TmaBoxMaps box_maps(const float* src, int W, int H, int planes) {
  TmaBoxMaps maps;
  for (int i = 0; i < TMA_BOX_HEIGHTS; ++i) maps.map[i] = emu::make_map(src, W, H, planes, BW, tma_box_rows(BH, i), 1);
  return maps;
}

template <bool PROJ, int PAD, int TW, int TH, int BW, int BH, int INTERP = KB200_BILINEAR, bool ALIGN = true>
static void test_forward(int B, int H, int W, int h, int w, unsigned grid, bool lazy, bool tame) {
  emu::lazy_tma = lazy;
  emu::set_smem(tma_smem, sizeof(tma_smem));
  constexpr int C = 3;
  const size_t ns = (size_t)B * C * H * W, no = (size_t)B * C * h * w;
  std::vector<float> ss, o1s, o2s;
  float* src = aligned(ss, ns);
  for (size_t i = 0; i < ns; ++i) src[i] = randv(1)[0];
  std::vector<float> m((size_t)B * 9), bx(w), by(h);
  for (int i = 0; i < w; ++i) bx[i] = ((float)i / (float)std::max(w - 1, 1) - 0.5f) * 2.f;
  for (int i = 0; i < h; ++i) by[i] = ((float)i / (float)std::max(h - 1, 1) - 0.5f) * 2.f;
  for (int b = 0; b < B; ++b) {
    const float t = tame ? 0.004f * (b - 1) : (b == 2 ? 0.436f : 0.02f * b);
    const float M[9] = {cosf(t) * (1.f + (tame ? 0.004f : 0.03f) * b), -sinf(t), (tame ? 0.01f : 0.05f) * b - (!tame && b == 1 ? 0.7f : 0.f), sinf(t),
                        cosf(t) * (tame ? 0.995f : 0.97f), tame ? -0.008f : -0.03f, PROJ ? (tame ? 0.004f : 0.02f) : 0.f, PROJ ? (tame ? -0.003f : -0.015f) : 0.f, 1.f};
    memcpy(&m[(size_t)b * 9], M, sizeof(M));
  }
  float* o1 = aligned(o1s, no);
  float* o2 = aligned(o2s, no);
  TmaWarpParams p{};
  const float fillc[3] = {0.25f, 0.5f, 0.75f};
  p.src = src; p.m = m.data(); p.bx = bx.data(); p.by = by.data(); p.fill = fillc;
  p.B = B; p.H = H; p.W = W; p.h = h; p.w = w; p.Bm = B; p.align = ALIGN ? 1 : 0; p.only_class = 0;
  // oracle: the exact per-pixel path of the same header (the generic kernel's arithmetic, verified against torch on hardware)
  p.out = o2;
  for (int b = 0; b < B; ++b)
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        const float* mm = &m[(size_t)b * 9];
        careful_pixel<C, INTERP, PAD, PROJ, ALIGN>(p, b, y, x, mm[0] * bx[x], mm[3] * bx[x], PROJ ? mm[6] * bx[x] : 0.f, mm[1] * by[y], mm[4] * by[y],
                                                          PROJ ? mm[7] * by[y] : 0.f, mm[2], mm[5], mm[8]);
      }
  p.out = o1;
  const TmaBoxMaps map = box_maps<BW, BH>(src, W, H, B * C);
  emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2>(map, p); });
  if (INTERP == KB200_BILINEAR && TW == 64) {  // the run-time work distribution: same tiles, same results
    std::vector<float> o3s;
    float* o3 = aligned(o3s, no);
    for (int chunk : {1, 3, 10}) {
      for (size_t i = 0; i < no; ++i) o3[i] = -5.f;
      int counter = 0;
      TmaWarpParams q = p;
      q.out = o3; q.counter = &counter; q.chunk_tiles = chunk; q.static_pct = chunk == 3 ? 50 : (chunk == 10 ? 100 : 0);
      emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2, true>(map, q); });
      p.out = o3;  // keep the comparison below on o1
      p.out = o1;
      compare("warp_fwd_tma<DYN> chunk=" + std::to_string(chunk) + " vs the static deal " + std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) +
                  " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"), o3, o2, no);
    }
    // the sweep: every run drawn in raster order (static_pct 0), runs of 1, 2 and 3 tiles; then the same launch restricted to the
    // footprint class of the wide tile (the producer skips the other class's samples and moves the counter past their runs)
    // against the static deal restricted the same way, with the rotated sample moved to the front twice so that two
    // consecutive samples are skipped
    std::vector<float> o4s, m2(m);
    float* o4 = aligned(o4s, no);
    if (B >= 3) {
      memcpy(&m2[0], &m[18], 9 * sizeof(float));
      memcpy(&m2[9], &m[18], 9 * sizeof(float));
      memcpy(&m2[18], &m[0], 9 * sizeof(float));
    }
    for (int run : {1, 2, 3}) {
      const std::string tag = " " + std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
      for (size_t i = 0; i < no; ++i) o3[i] = -5.f;
      int counter = 0;
      TmaWarpParams q = p;
      q.out = o3; q.counter = &counter; q.chunk_tiles = run; q.static_pct = 0;
      emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2, true>(map, q); });
      compare("warp_fwd_tma<DYN> sweep run=" + std::to_string(run) + " vs its exact path" + tag, o3, o2, no);
      for (size_t i = 0; i < no; ++i) o3[i] = o4[i] = -5.f;
      counter = 0;
      q.only_class = CLASS_WIDE; q.m = m2.data();
      emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2, true>(map, q); });
      TmaWarpParams r = p;
      r.out = o4; r.only_class = CLASS_WIDE; r.m = m2.data();
      emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2>(map, r); });
      compare("warp_fwd_tma<DYN> sweep run=" + std::to_string(run) + " wide class only vs the static deal" + tag, o3, o4, no);
    }
  }
  compare(std::string("warp_fwd_tma (headline, verified on hw) vs its exact path ") + (PROJ ? "projective " : "affine ") + "interp=" + std::to_string(INTERP) + " pad=" + std::to_string(PAD) + " tile " +
              std::to_string(TW) + "x" + std::to_string(TH) + " " + std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) + " -> " + std::to_string(h) +
              "x" + std::to_string(w) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager") + (tame ? " tame" : " wild") + (ALIGN ? "" : " align_corners=False"),
          o1, o2, no);
}

// ------------------------------------------------------------------------------------------ tiled warp backward
template <bool PROJ>
static void test_backward(int B, int H, int W, int h, int w, unsigned grid, bool lazy, bool tame = false) {
  emu::lazy_tma = lazy;
  constexpr int C = 3;
  constexpr bool ALIGN = true;
  const size_t ns = (size_t)B * C * H * W, no = (size_t)B * C * h * w;
  std::vector<float> ss, gs, g1s, g2s;
  float* src = aligned(ss, ns);
  float* gout = aligned(gs, no);
  for (size_t i = 0; i < ns; ++i) src[i] = randv(1)[0];
  for (size_t i = 0; i < no; ++i) gout[i] = randv(1, -0.5f, 0.5f)[0];
  std::vector<float> m((size_t)B * 9), bx(w), by(h);
  for (int i = 0; i < w; ++i) bx[i] = ((float)i / (float)(w - 1) - 0.5f) * 2.f;
  for (int i = 0; i < h; ++i) by[i] = ((float)i / (float)(h - 1) - 0.5f) * 2.f;
  for (int b = 0; b < B; ++b) {  // normalised src <- dst maps: near identity, a shift out of view, a 25 degree rotation
    // tame: the headline's kind of map (a few pixels of jitter): almost every pixel on the shared-memory fast path
    const float t = tame ? 0.004f * (b - 1) : (b == 2 ? 0.436f : 0.02f * b);
    const float M[9] = {cosf(t) * (1.f + (tame ? 0.004f : 0.03f) * b), -sinf(t), (tame ? 0.01f : 0.05f) * b - (!tame && b == 1 ? 0.7f : 0.f), sinf(t),
                        cosf(t) * (tame ? 0.995f : 0.97f), tame ? -0.008f : -0.03f, PROJ ? (tame ? 0.004f : 0.02f) : 0.f, PROJ ? (tame ? -0.003f : -0.015f) : 0.f, 1.f};
    memcpy(&m[(size_t)b * 9], M, sizeof(M));
  }
  // scalar reference in double (same fp32 coordinate chain through the kernels' own helpers)
  std::vector<double> gsrc_ref(ns, 0.0), gm_ref((size_t)B * 9, 0.0);
  const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1);
  for (int b = 0; b < B; ++b) {
    Mat3<float> mm;
    mm.load(&m[(size_t)b * 9]);
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        float gx, gy, den;
        map_point<float, PROJ>(mm, bx[x], by[y], gx, gy, den);
        const float ix = unnorm<ALIGN>(gx, Wm1, (float)W), iy = unnorm<ALIGN>(gy, Hm1, (float)H);
        if (!(fabsf(ix) < 1.0e9f && fabsf(iy) < 1.0e9f)) continue;
        const float x0f = floorf(ix), y0f = floorf(iy);
        const double wx1 = (double)((x0f + 1.f) - ix), wx0 = (double)(ix - x0f), wy1 = (double)((y0f + 1.f) - iy), wy0 = (double)(iy - y0f);
        const int x0 = (int)x0f, y0 = (int)y0f;
        double gix = 0, giy = 0;
        for (int c = 0; c < C; ++c) {
          const double go = gout[(((size_t)b * C + c) * h + y) * w + x];
          const float* sp = src + ((size_t)b * C + c) * H * W;
          double* gp = gsrc_ref.data() + ((size_t)b * C + c) * H * W;
          auto ok = [&](int yy, int xx) { return yy >= 0 && yy < H && xx >= 0 && xx < W; };
          auto v = [&](int yy, int xx) { return ok(yy, xx) ? (double)sp[(size_t)yy * W + xx] : 0.0; };
          if (ok(y0, x0)) gp[(size_t)y0 * W + x0] += wx1 * wy1 * go;
          if (ok(y0, x0 + 1)) gp[(size_t)y0 * W + x0 + 1] += wx0 * wy1 * go;
          if (ok(y0 + 1, x0)) gp[(size_t)(y0 + 1) * W + x0] += wx1 * wy0 * go;
          if (ok(y0 + 1, x0 + 1)) gp[(size_t)(y0 + 1) * W + x0 + 1] += wx0 * wy0 * go;
          gix += go * ((v(y0, x0 + 1) - v(y0, x0)) * wy1 + (v(y0 + 1, x0 + 1) - v(y0 + 1, x0)) * wy0);
          giy += go * ((v(y0 + 1, x0) - v(y0, x0)) * wx1 + (v(y0 + 1, x0 + 1) - v(y0, x0 + 1)) * wx0);
        }
        const double rden = PROJ ? 1.0 / (double)den : 1.0;
        const double ax = gix * (Wm1 * 0.5) * rden, ay = giy * (Hm1 * 0.5) * rden, az = -(ax * gx + ay * gy);
        double* g = &gm_ref[(size_t)b * 9];
        g[0] += ax * bx[x]; g[1] += ax * by[y]; g[2] += ax;
        g[3] += ay * bx[x]; g[4] += ay * by[y]; g[5] += ay;
        if (PROJ) { g[6] += az * bx[x]; g[7] += az * by[y]; g[8] += az; }
      }
  }
  const int nstrips = B * ceil_div(h, 32), max_segs = nstrips / (int)grid + 2;
  const size_t rows = (size_t)grid * max_segs;
  long long exact[6] = {0, 0, 0, 0, 0, 0};
  auto run = [&](int version, float* gsrc, std::vector<double>& gm) {
    emu_exact_path_pixels = 0;
    for (size_t i = 0; i < ns; ++i) gsrc[i] = 0.f;
    std::vector<float> records(rows * 8 * 9, 0.f);
    std::vector<int> rb(rows, -7);
    TmaBwdParams p{};
    p.gout = gout; p.src = src; p.m = m.data(); p.bx = bx.data(); p.by = by.data(); p.gsrc = gsrc;
    p.records = records.data(); p.record_batch = rb.data();
    p.B = B; p.H = H; p.W = W; p.h = h; p.w = w; p.Bm = B; p.max_segs = max_segs;
    const CUtensorMap mgsrc = emu::make_map(gsrc, W, H, B * C, 72, BWD_SH, C), mgout = emu::make_map(gout, w, h, B * C, 64, 32, C);
    emu::set_smem(bwd2_smem, sizeof(bwd2_smem));
    const CUtensorMap mwin = emu::make_map(src, W, H, B * C, 72, BWD_SH, C);
    int counter = 0;
    size_t use_rows = rows;
    if (version == 5) {  // the run-time work distribution: one record row per chunk, chunk = 3 tiles here
      p.counter = &counter;
      p.chunk_tiles = 3;
      use_rows = (size_t)B * ceil_div(h, 32) * ceil_div(ceil_div(w, 64), 3);
      records.assign(use_rows * 8 * 9, 0.f);
      rb.assign(use_rows, -7);
      p.records = records.data(); p.record_batch = rb.data();
      emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, KB200_ZEROS, PROJ, ALIGN, true, true, true, true>(mwin, mgsrc, mgout, p); });
    } else
    if (version == 2) emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, KB200_ZEROS, PROJ, ALIGN, true, true, false>(mwin, mgsrc, mgout, p); });
    else emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, KB200_ZEROS, PROJ, ALIGN, true, true, true>(mwin, mgsrc, mgout, p); });
    exact[version] = emu_exact_path_pixels;
    gm.assign((size_t)B * 9, 0.0);
    for (size_t r = 0; r < use_rows; ++r)
      if (rb[r] >= 0)
        for (int wv = 0; wv < 8; ++wv)
          for (int k = 0; k < 9; ++k) gm[(size_t)rb[r] * 9 + k] += (double)records[(r * 8 + wv) * 9 + k];
  };
  const std::string tag = std::string(PROJ ? "projective " : "affine     ") + std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) + " -> " +
                          std::to_string(h) + "x" + std::to_string(w) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
  float* g1 = aligned(g1s, ns);
  float* g2 = aligned(g2s, ns);
  std::vector<double> gm1, gm2;
  std::vector<float> g5s;
  float* g5 = aligned(g5s, ns);
  std::vector<double> gm5;
  run(2, g1, gm1);
  run(3, g2, gm2);
  run(5, g5, gm5);
  auto check = [&](const char* name, const float* g, const std::vector<double>& gm) {
    double num = 0, den = 0, worst = 0;
    for (size_t i = 0; i < ns; ++i) {
      const double d = (double)g[i] - gsrc_ref[i];
      num += d * d; den += gsrc_ref[i] * gsrc_ref[i];
      worst = std::max(worst, fabs(d));
    }
    double mn = 0, md = 0;
    for (size_t i = 0; i < gm.size(); ++i) { mn += (gm[i] - gm_ref[i]) * (gm[i] - gm_ref[i]); md += gm_ref[i] * gm_ref[i]; }
    const double e_src = sqrt(num / den), e_m = sqrt(mn / md);
    const bool ok = e_src < 2e-6 && worst < 2e-5 && e_m < 1e-4;
    printf("%s %-58s %s  d/dsrc rel-L2 %.2e max-abs %.2e, d/dM rel-L2 %.2e\n", ok ? "ok  " : "FAIL", name, tag.c_str(), e_src, worst, e_m);
    if (!ok) ++failures;
  };
  printf("     pixels on the exact (global-memory) path: warp_bwd_tma2 %lld, stride-1 lanes %lld of %d\n", exact[2], exact[3], B * h * w);
  check("warp_bwd_tma2 (per-warp pipelines) vs fp64 scalar backward", g1, gm1);
  check("warp_bwd_tma2<STRIDE1> (conflict-free lanes) vs fp64 scalar backward", g2, gm2);
  check("warp_bwd_tma2<STRIDE1, DYN> (work drawn at run time) vs fp64 scalar backward", g5, gm5);
}

// Random shapes, grids and completion modes (run_emu --fuzz N): shakes out the edge cases the fixed list does not name
// -- images smaller than a tile, one-row last tiles, bands narrower than the halo, more CTAs than strips.
// ------------------------------------------------------------------------------------------ uint8 ingest warp
// warp_fwd_u8hwc on interleaved bytes against the hardware-verified generic kernel on the planar fp32 image the
// reference would have built first (io.py:111 as torch evaluates it: a real division on CPU, times 1.0f / 255.0f on CUDA): bit for bit.
template <int INTERP, int PAD, int KIND>
static void test_u8(int B, int C, int H, int W, int h, int w, bool align, int normalize, bool shared_m) {
  const size_t npix = (size_t)B * H * W, no = (size_t)B * C * h * w;
  std::vector<unsigned char> bytes(npix * C);
  for (auto& v : bytes) v = (unsigned char)(rng() & 255);
  std::vector<float> planar(npix * C), o1(no, -1.f), o2(no, -2.f), m((size_t)B * 9), bx(w), by(h);
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c)
      for (int i = 0; i < H * W; ++i) {
        const float f = (float)bytes[((size_t)b * H * W + i) * C + c];
        planar[((size_t)b * C + c) * H * W + i] = normalize == 2 ? f / 255.0f : normalize == 1 ? f * (1.0f / 255.0f) : f;
      }
  for (int i = 0; i < w; ++i) bx[i] = ((float)i / (float)std::max(w - 1, 1) - 0.5f) * 2.f;
  for (int i = 0; i < h; ++i) by[i] = ((float)i / (float)std::max(h - 1, 1) - 0.5f) * 2.f;
  for (int b = 0; b < B; ++b) {
    const float t = 0.3f * b - 0.2f;
    const float M[9] = {cosf(t) * (1.f + 0.1f * b), -sinf(t), 0.2f * b - 0.3f, sinf(t), cosf(t) * 0.9f, 0.15f,
                        KIND == KIND_PROJ ? 0.05f : 0.f, KIND == KIND_PROJ ? -0.04f : 0.f, 1.f};
    memcpy(&m[(size_t)b * 9], M, sizeof(M));
  }
  const float fillc[4] = {0.25f, 0.5f, 0.75f, 1.f};
  const int Bm = shared_m ? 1 : B;
  WarpParams<float> g{};
  g.src = planar.data(); g.m = m.data(); g.bx = bx.data(); g.by = by.data(); g.fill = fillc; g.out = o2.data();
  g.B = B; g.C = C; g.H = H; g.W = W; g.h = h; g.w = w; g.Bm = Bm; g.align = align; g.normalized = 0;
  WarpU8Params u{};
  u.src = bytes.data(); u.m = m.data(); u.bx = bx.data(); u.by = by.data(); u.fill = fillc; u.out = o1.data();
  u.B = B; u.C = C; u.H = H; u.W = W; u.h = h; u.w = w; u.Bm = Bm; u.align = align; u.normalize = normalize;
  const dim3 grid(ceil_div(w, GEN_BX), ceil_div(h, GEN_BY), B), block(GEN_BX, GEN_BY);
  emu::launch3(grid, block, [&] { warp_fwd_generic<float, INTERP, PAD, KIND>(g); });
  if (C == 3)  // the instantiation the host picks (warp_u8.cu:launch_u8)
    emu::launch3(grid, block, [&] { warp_fwd_u8hwc<INTERP, PAD, KIND, 3>(u); });
  else if (C == 1)
    emu::launch3(grid, block, [&] { warp_fwd_u8hwc<INTERP, PAD, KIND, 1>(u); });
  else
    emu::launch3(grid, block, [&] { warp_fwd_u8hwc<INTERP, PAD, KIND, 0>(u); });
  compare("warp_fwd_u8hwc vs convert + warp_fwd_generic interp=" + std::to_string(INTERP) + " pad=" + std::to_string(PAD) + " kind=" + std::to_string(KIND) + " " +
              std::to_string(B) + "x" + std::to_string(H) + "x" + std::to_string(W) + "x" + std::to_string(C) + " -> " + std::to_string(h) + "x" + std::to_string(w) +
              (align ? " align" : "") + (normalize == 2 ? " /255" : normalize == 1 ? " *(1/255)" : " raw") + (shared_m ? " shared matrix" : ""),
          o1.data(), o2.data(), no);
}

// warp_u8_tiled_kernel (cooperative byte staging, every byte converted once) against warp_fwd_u8hwc (per-tap conversion):
// bit for bit, on maps that keep most pixels on the shared-memory path (tame) and on maps that push tiles to the exact path.
template <int NC, int PAD, bool PROJ, bool ALIGN>
static void test_u8_tiled(int B, int H, int W, int h, int w, int normalize, bool tame, bool shared_m, bool check_share = true) {
  emu::set_smem(u8t_smem, sizeof(u8t_smem));
  const size_t npix = (size_t)B * H * W, no = (size_t)B * NC * h * w;
  std::vector<unsigned char> store(npix * NC + 64);
  unsigned char* bytes = store.data() + ((4 - (reinterpret_cast<uintptr_t>(store.data()) & 3)) & 3);  // 4-byte aligned, as the host requires
  for (size_t i = 0; i < npix * NC; ++i) bytes[i] = (unsigned char)(rng() & 255);
  std::vector<float> o1(no, -1.f), o2(no, -2.f), m((size_t)B * 9), bx(w), by(h);
  for (int i = 0; i < w; ++i) bx[i] = ALIGN || !PROJ ? ((float)i / (float)std::max(w - 1, 1) - 0.5f) * 2.f : ((float)i / (float)std::max(w - 1, 1) - 0.5f) * 2.f;
  for (int i = 0; i < h; ++i) by[i] = ((float)i / (float)std::max(h - 1, 1) - 0.5f) * 2.f;
  for (int b = 0; b < B; ++b) {
    const float t = tame ? 0.01f * (b - 1) : 0.5f * b - 0.3f;
    const float M[9] = {cosf(t) * (tame ? 1.01f : 1.3f), -sinf(t), tame ? 0.02f * b : 0.4f * b - 0.5f, sinf(t), cosf(t) * (tame ? 0.99f : 0.8f), tame ? -0.01f : 0.3f,
                        PROJ ? (tame ? 0.004f : 0.08f) : 0.f, PROJ ? (tame ? -0.003f : -0.06f) : 0.f, 1.f};
    memcpy(&m[(size_t)b * 9], M, sizeof(M));
  }
  WarpU8Params u{};
  static const float fillc[4] = {0.25f, 0.5f, 0.75f, 1.0f};
  u.src = bytes; u.m = m.data(); u.bx = bx.data(); u.by = by.data(); u.fill = fillc;
  u.B = B; u.C = NC; u.H = H; u.W = W; u.h = h; u.w = w; u.Bm = shared_m ? 1 : B; u.align = ALIGN; u.normalize = normalize;
  u.out = o2.data();
  emu::launch3(dim3(ceil_div(w, GEN_BX), ceil_div(h, GEN_BY), B), dim3(GEN_BX, GEN_BY),
               [&] { warp_fwd_u8hwc<KB200_BILINEAR, PAD, PROJ ? KIND_PROJ : KIND_AFFINE, NC>(u); });
  u.out = o1.data();
  u8t_fast_pixels = u8t_exact_pixels = 0;
  emu::launch3(dim3(ceil_div(w, 64), ceil_div(h, 32), B), dim3(256), [&] { warp_u8_tiled_kernel<NC, PAD, PROJ ? KIND_PROJ : KIND_AFFINE, ALIGN>(u); });
  const int fast_pct = (int)(100 * u8t_fast_pixels / std::max(1ll, u8t_fast_pixels + u8t_exact_pixels));
  if (tame && check_share && fast_pct < 50) {
    ++failures;
    printf("FAIL warp_u8_tiled_kernel: only %d %% of the pixels of a near-identity map took the shared-memory path\n", fast_pct);
  }
  compare(std::string("warp_u8_tiled_kernel vs warp_fwd_u8hwc ") + (PROJ ? "projective" : "affine") + " pad=" + std::to_string(PAD) + " " + std::to_string(B) + "x" +
              std::to_string(H) + "x" + std::to_string(W) + "x" + std::to_string(NC) + " -> " + std::to_string(h) + "x" + std::to_string(w) + (ALIGN ? " align" : "") +
              " normalize=" + std::to_string(normalize) + (tame ? " tame" : " wild") + (shared_m ? " shared matrix" : "") + ", " + std::to_string(fast_pct) + " % from shared memory",
          o1.data(), o2.data(), no);
}

// undistort_image from decoder bytes (warp_u8_tiled_kernel<U8_KIND_LENS>) against the fp32 fused undistort
// (remap_tiled_kernel<LENS>, itself checked against maps + remap above) on the image the reference would have converted first.
template <int NC>
static void test_u8_undistort(int B, int H, int W, int normalize, bool strong) {
  const size_t npix = (size_t)B * H * W, n = npix * NC;
  std::vector<unsigned char> store(n + 64);
  unsigned char* bytes = store.data() + ((4 - (reinterpret_cast<uintptr_t>(store.data()) & 3)) & 3);
  for (size_t i = 0; i < n; ++i) bytes[i] = (unsigned char)(rng() & 255);
  std::vector<float> ss, o1(n, -1.f), o2(n, -2.f), lens((size_t)B * 16);
  float* planar = aligned(ss, n);
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < NC; ++c)
      for (int i = 0; i < H * W; ++i) {
        const float f = (float)bytes[((size_t)b * H * W + i) * NC + c];
        planar[((size_t)b * NC + c) * H * W + i] = normalize == 2 ? f / 255.0f : normalize == 1 ? f * (1.0f / 255.0f) : f;
      }
  for (int b = 0; b < B; ++b) {
    const float L[16] = {(strong ? 0.35f : 0.8f) * W + 3 * b, (strong ? 0.3f : 0.75f) * W, 0.5f * W - 3.f, 0.5f * H + 2.f, strong ? -0.45f : -0.21f, 0.07f, 0.002f, -0.003f, 0.01f, 0.04f, -0.02f, 0.004f, 0.003f, -0.001f, 0.002f, 0.0015f};
    memcpy(&lens[(size_t)b * 16], L, sizeof(L));
  }
  const dim3 grid(ceil_div(W, 64), ceil_div(H, 32), B);
  emu::lazy_tma = false;
  emu::set_smem(remap_smem, sizeof(remap_smem));
  const CUtensorMap map = emu::make_map(planar, W, H, B * NC, 72, 40, NC);
  RemapTiledParams rp{planar, nullptr, nullptr, o2.data(), B, H, W, H, W, B, 0, lens.data()};
  emu::launch3(grid, dim3(256), [&] { remap_tiled_kernel<NC, KB200_ZEROS, true, true>(map, rp); });
  emu::set_smem(u8t_smem, sizeof(u8t_smem));
  WarpU8Params u{};
  u.src = bytes; u.lens = lens.data(); u.out = o1.data();
  u.B = B; u.C = NC; u.H = H; u.W = W; u.h = H; u.w = W; u.Bm = B; u.align = 1; u.normalize = normalize;
  u8t_fast_pixels = u8t_exact_pixels = 0;
  emu::launch3(grid, dim3(256), [&] { warp_u8_tiled_kernel<NC, KB200_ZEROS, U8_KIND_LENS, true>(u); });
  compare("warp_u8_tiled_kernel<LENS> (undistort from bytes) vs convert + remap_tiled_kernel<LENS> " + std::to_string(B) + "x" + std::to_string(H) + "x" +
              std::to_string(W) + "x" + std::to_string(NC) + " normalize=" + std::to_string(normalize) + (strong ? " strong" : "") + ", " +
              std::to_string((int)(100 * u8t_fast_pixels / std::max(1ll, u8t_fast_pixels + u8t_exact_pixels))) + " % from shared memory",
          o1.data(), o2.data(), n);
}

static void test_u8_all() {
  int bad = 0;
  for (int v = 0; v < 256; ++v) bad += unit_from_byte((unsigned char)v) != (float)v / 255.0f;
  for (int v = 0; v < 256; ++v) bad += level_of_byte((unsigned char)v) != (float)v;
  for (int v = 0; v < 256; ++v)  // the PRMT + FADD conversion of the tiled loader, every byte in every lane of a word
    for (int q = 0; q < 4; ++q) bad += level_of_word_byte(0xA5C3E17Bu ^ (((unsigned)v ^ ((0xA5C3E17Bu >> (8 * q)) & 255u)) << (8 * q)), q) != (float)v;
  if (bad) {
    ++failures;
    printf("FAIL unit_from_byte: %d of 256 bytes differ from float(u) / 255.0f\n", bad);
  } else {
    printf("ok   unit_from_byte == float(u) / 255.0f for all 256 bytes\n");
  }
  test_u8<KB200_BILINEAR, KB200_ZEROS, KIND_PROJ>(2, 3, 37, 52, 37, 52, true, 1, false);
  test_u8<KB200_BILINEAR, KB200_BORDER, KIND_PROJ>(2, 3, 37, 52, 29, 61, false, 2, false);
  test_u8<KB200_BILINEAR, KB200_REFLECTION, KIND_AFFINE>(3, 1, 20, 33, 41, 35, true, 2, true);
  test_u8<KB200_BILINEAR, KB200_FILL, KIND_PROJ>(2, 3, 37, 52, 37, 52, true, 1, false);
  test_u8<KB200_NEAREST, KB200_ZEROS, KIND_PROJ>(2, 4, 18, 26, 30, 30, false, 0, false);
  test_u8<KB200_NEAREST, KB200_FILL, KIND_AFFINE>(1, 3, 18, 26, 18, 26, true, 1, false);
  test_u8<KB200_BICUBIC, KB200_ZEROS, KIND_PROJ>(2, 3, 37, 52, 37, 52, true, 1, false);
  test_u8<KB200_BICUBIC, KB200_REFLECTION, KIND_AFFINE>(2, 4, 19, 23, 33, 40, false, 2, false);
  test_u8<KB200_BICUBIC, KB200_FILL, KIND_PROJ>(1, 3, 16, 16, 20, 24, true, 0, false);
  test_u8_tiled<3, KB200_ZEROS, true, true>(3, 70, 132, 70, 132, 1, true, false);
  test_u8_tiled<3, KB200_ZEROS, true, true>(3, 70, 132, 50, 100, 1, false, false);
  test_u8_tiled<3, KB200_BORDER, true, false>(2, 64, 128, 70, 132, 2, true, false);
  test_u8_tiled<3, KB200_REFLECTION, false, true>(3, 40, 76, 66, 130, 1, true, true);
  test_u8_tiled<3, KB200_REFLECTION, true, true>(2, 70, 132, 70, 132, 0, false, false);
  test_u8_tiled<1, KB200_ZEROS, false, false>(3, 70, 132, 96, 200, 1, true, false);
  test_u8_tiled<1, KB200_BORDER, true, true>(2, 33, 64, 40, 70, 2, false, false);
  test_u8_tiled<1, KB200_REFLECTION, false, true>(2, 9, 8, 20, 24, 1, true, false);
  test_u8_tiled<3, KB200_ZEROS, false, true>(2, 5, 4, 33, 65, 1, true, false);
  test_u8_tiled<3, KB200_FILL, true, true>(3, 70, 132, 70, 132, 1, true, false);
  test_u8_tiled<3, KB200_FILL, true, false>(2, 40, 76, 66, 130, 2, false, false);
  test_u8_tiled<1, KB200_FILL, false, true>(2, 33, 64, 40, 70, 0, true, true);
  test_u8_tiled<4, KB200_ZEROS, true, true>(2, 70, 132, 70, 132, 1, true, false);
  test_u8_tiled<4, KB200_FILL, false, false>(2, 33, 64, 40, 70, 2, false, false);
  test_u8_tiled<4, KB200_REFLECTION, true, true>(1, 40, 76, 66, 130, 0, true, false);
  test_u8_undistort<3>(2, 70, 132, 1, false);
  test_u8_undistort<3>(2, 97, 200, 2, true);
  test_u8_undistort<1>(1, 33, 64, 0, false);
}


// reflect_clip_near_rt (two subtractions and a select) against clip_coord(reflect_coord(...)) (fmod, division, floor): every float
// within 300 ulps of a multiple of the span and a random sweep of +-3 spans, for several sizes and both align_corners settings.
static void test_reflect_near() {
  long long checked = 0, bad = 0, fars = 0;
  std::mt19937 g(7);
  for (int size : {1, 2, 3, 5, 64, 720, 1080, 1920, 4099})
    for (int align = 0; align < 2; ++align) {
      const int tl = align ? 0 : -1, th = align ? 2 * (size - 1) : 2 * size - 1;
      const float lo = tl * 0.5f, span = (th - tl) * 0.5f;
      auto check = [&](float c) {
        bool far = false;
        const float got = reflect_clip_near_rt<float>(c, size, align != 0, far);
        const float want = clip_coord(reflect_coord(c, tl, th), size);
        ++checked;
        if (far) { ++fars; return; }
        bool far2 = false;  // idempotent: padding the padded coordinate again returns it (the pipelined remap relies on it)
        const float again = reflect_clip_near_rt<float>(got, size, align != 0, far2);
        if (far2 || (memcmp(&again, &got, 4) != 0 && !(again == 0.f && got == 0.f))) {
          if (bad < 5) printf("     reflect not idempotent size=%d align=%d c=%.9g first %.9g second %.9g\n", size, align, c, got, again);
          ++bad;
        }
        if (memcmp(&got, &want, 4) != 0 && !(got == 0.f && want == 0.f)) {
          if (bad < 5) printf("     reflect mismatch size=%d align=%d c=%.9g got %.9g want %.9g\n", size, align, c, got, want);
          ++bad;
        }
      };
      for (int k = -3; k <= 3; ++k) {
        float c = lo + k * span;
        for (int i = 0; i < 300; ++i) c = nextafterf(c, -INFINITY);
        for (int i = 0; i < 600; ++i, c = nextafterf(c, INFINITY)) check(c);
      }
      for (int i = 0; i < 20000; ++i) check(lo + ((float)(g() % 2000001) / 1000000.f - 1.f) * 3.f * std::max(span, 1.f));
      check(NAN); check(INFINITY); check(-INFINITY); check(1e30f);
    }
  printf("%s reflect_clip_near_rt == clip_coord(reflect_coord) on %lld coordinates (%lld beyond two spans left to the general form)\n", bad ? "FAIL" : "ok  ",
         checked, fars);
  if (bad) ++failures;
}

// run_emu --probe PAD: one 540 x 960 sample under a bench-like homography (a few pixels of shift, 1 % scale): how many tiles run
// the INNER copy and how many pixels leave the shared-memory path, per padding mode.
template <int PAD, int INTERP = KB200_BILINEAR>
static void probe_forward() {
  constexpr int C = 3, H = 540, W = 960;
  emu::lazy_tma = false;
  emu::set_smem(tma_smem, sizeof(tma_smem));
  std::vector<float> ss, o1s;
  float* src = aligned(ss, (size_t)C * H * W);
  for (size_t i = 0; i < (size_t)C * H * W; ++i) src[i] = randv(1)[0];
  std::vector<float> bx(W), by(H);
  for (int i = 0; i < W; ++i) bx[i] = ((float)i / (float)(W - 1) - 0.5f) * 2.f;
  for (int i = 0; i < H; ++i) by[i] = ((float)i / (float)(H - 1) - 0.5f) * 2.f;
  const float M[9] = {1.0013f, 0.0006f, -4.24f * 2.f / (W - 1), 0.0015f, 1.0155f, -9.04f * 2.f / (H - 1), 0.001f, 0.0004f, 1.f};
  float* o1 = aligned(o1s, (size_t)C * H * W);
  TmaWarpParams p{};
  const float fillc[3] = {0.25f, 0.5f, 0.75f};
  p.src = src; p.m = M; p.bx = bx.data(); p.by = by.data(); p.fill = fillc; p.out = o1;
  p.B = 1; p.H = H; p.W = W; p.h = H; p.w = W; p.Bm = 1; p.align = 1; p.only_class = 0;
  const TmaBoxMaps map = box_maps<72, 40>(src, W, H, C);
  emu_careful_pixels = emu_inner_tiles = emu_other_tiles = 0;
  emu::launch(4, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, true, true, 64, 32, 72, 40, 2>(map, p); });
  printf("interp=%d pad=%d: tiles INNER %lld other %lld (each counted once per CTA), pixels on the exact path %lld of %d\n", INTERP, PAD, emu_inner_tiles, emu_other_tiles,
         emu_careful_pixels, H * W);
}

static void fuzz(int rounds) {
  std::mt19937 g(20260923);
  auto pick = [&](int lo, int hi) { return lo + (int)(g() % (unsigned)(hi - lo + 1)); };
  for (int r = 0; r < rounds; ++r) {
    const int H = pick(1, 110), W = 4 * pick(1, 70), planes = pick(1, 4), lazy = pick(0, 1);
    const unsigned grid = (unsigned)pick(1, 9);
    switch (pick(0, 40)) {
      case 35: if (H > 1) test_forward<true, KB200_BORDER, 64, 32, 72, 40, KB200_BICUBIC, false>(3, H, W, std::max(1, H - pick(0, 5)), std::max(4, W - 4 * pick(0, 3)), grid, lazy, pick(0, 1)); break;
      case 36: if (H > 1) test_forward<true, KB200_REFLECTION, 64, 32, 72, 40, KB200_BICUBIC, true>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 37: if (H > 1) test_forward<false, KB200_REFLECTION, 64, 32, 72, 40, KB200_BICUBIC, false>(3, H, W, std::max(1, H - pick(0, 5)), W, grid, lazy, pick(0, 1)); break;
      case 38: if (H > 1) test_forward<true, KB200_FILL, 64, 32, 72, 40, KB200_BICUBIC, true>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 39: if (H > 1) test_forward<false, KB200_FILL, 32, 32, 56, 56, KB200_BICUBIC, false>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 40: if (H > 1) test_forward<true, KB200_BORDER, 32, 32, 56, 56, KB200_BICUBIC, true>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 25: if (H > 1) test_forward<true, KB200_REFLECTION, 64, 32, 72, 40, KB200_BILINEAR, false>(3, H, W, std::max(1, H - pick(0, 5)), std::max(4, W - 4 * pick(0, 3)), grid, lazy, pick(0, 1)); break;
      case 26: if (H > 1) test_forward<true, KB200_FILL, 64, 32, 72, 40, KB200_BILINEAR, false>(3, H, W, std::max(1, H - pick(0, 5)), std::max(4, W - 4 * pick(0, 3)), grid, lazy, pick(0, 1)); break;
      case 27: if (H > 1) test_forward<false, KB200_REFLECTION, 64, 32, 72, 40, KB200_NEAREST, true>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 28: if (H > 1) test_forward<true, KB200_FILL, 64, 32, 72, 40, KB200_NEAREST, false>(3, H, W, std::max(1, H - pick(0, 5)), W, grid, lazy, pick(0, 1)); break;
      case 29: if (H > 1) test_forward<true, KB200_REFLECTION, 32, 32, 56, 56, KB200_BILINEAR, true>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 30: if (H > 1) test_forward<false, KB200_FILL, 64, 32, 72, 40, KB200_BILINEAR, true>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 10: if (H > 1 && W > 1) test_filter2d<3, KB200_REFLECT>(planes, H, W, grid, lazy); break;
      case 11: if (H > 3 && W > 3) test_filter2d<7, KB200_REPLICATE>(planes, H, W, grid, lazy); break;
      case 12: test_filter2d<7, KB200_CONSTANT>(planes, H, W, grid, lazy); break;
      case 13: if (H > 1) test_undistort(pick(1, 2), H, W, lazy); break;
      case 14: if (H > 1 && W > 4) test_backward<true>(3, H, W, std::max(2, H - pick(0, 3)), std::max(8, W - 4 * pick(0, 2)), grid, lazy, pick(0, 1)); break;
      case 16: if (H > 1) test_forward<true, KB200_ZEROS, 64, 32, 72, 40>(3, H, W, std::max(1, H - pick(0, 5)), std::max(4, W - 4 * pick(0, 3)), grid, lazy, pick(0, 1)); break;
      case 17: if (H > 1) test_forward<false, KB200_BORDER, 32, 32, 56, 56>(3, H, W, H, W, grid, lazy, pick(0, 1)); break;
      case 15: if (H > 1 && W > 4) test_backward<false>(3, std::max(2, H - 1), W, H, W, grid, lazy, true); break;
      case 18: test_u8_tiled<3, KB200_ZEROS, true, true>(pick(1, 3), H, W, std::max(1, H - pick(0, 5)), std::max(1, W - pick(0, 9)), pick(0, 2), pick(0, 1), false, false); break;
      case 19: test_u8_tiled<3, KB200_BORDER, false, false>(pick(1, 3), H, W, pick(1, 80), pick(1, 150), pick(0, 2), pick(0, 1), pick(0, 1), false); break;
      case 20: test_u8_tiled<1, KB200_REFLECTION, true, false>(pick(1, 3), H, W, H, W, pick(0, 2), pick(0, 1), false, false); break;
      case 21: test_u8_tiled<3, KB200_REFLECTION, true, true>(pick(1, 2), H, W, std::max(1, H - pick(0, 5)), W, pick(0, 2), pick(0, 1), false, false); break;
      case 23: test_u8_tiled<3, KB200_FILL, true, true>(pick(1, 2), H, W, std::max(1, H - pick(0, 5)), std::max(1, W - pick(0, 9)), pick(0, 2), pick(0, 1), false, false); break;
      case 24: test_u8_tiled<4, KB200_BORDER, true, false>(pick(1, 2), H, W, std::max(1, H - pick(0, 5)), std::max(1, W - pick(0, 9)), pick(0, 2), pick(0, 1), false, false); break;
      case 22: if (H > 1) test_u8_undistort<3>(pick(1, 2), H, W, pick(0, 2), pick(0, 1)); break;
      case 0: if (H > 5 && W > 5) test_sepfilter<11, KB200_REFLECT>(1, planes, H, W, grid, lazy); break;
      case 1: if (H > 8 && W > 8) test_sepfilter<17, KB200_REPLICATE>(1, planes, H, W, grid, lazy); break;
      case 2: test_sepfilter<5, KB200_CONSTANT>(planes, 1, H, W, grid, lazy); break;
      case 3: if (H > 1 && W > 1) test_sepfilter<3, KB200_REFLECT>(1, planes, H, W, grid, lazy); break;
      case 4: if (H > 2) test_pyrdown<KB200_REFLECT>(planes, 2 * ((H + 1) / 2) + 2, W, grid, lazy); break;
      case 5: test_pyrdown<KB200_CONSTANT>(planes, 2 * ((H + 1) / 2), W, grid, lazy); break;
      case 6: if (H > 2) test_gradient<5, 3, false>(planes, H, W, grid, lazy); break;
      case 7: if (H > 1) test_gradient<3, 2, true>(planes, H, W, grid, lazy); break;
      case 8: if (H > 5 && W > 5) test_ssim<11>(planes, H, W, grid, lazy); break;
      default: if (H > 3 && W > 3) test_ssim<7>(planes, H, W, grid, lazy); break;
    }
  }
}

int main(int argc, char** argv) {
  if (argc == 2 && std::string(argv[1]) == "--probe") {
    probe_forward<KB200_ZEROS>();
    probe_forward<KB200_BORDER>();
    probe_forward<KB200_REFLECTION>();
    probe_forward<KB200_ZEROS, KB200_BICUBIC>();
    probe_forward<KB200_BORDER, KB200_BICUBIC>();
    probe_forward<KB200_REFLECTION, KB200_BICUBIC>();
    probe_forward<KB200_FILL, KB200_BICUBIC>();
    return 0;
  }
  if (argc == 3 && std::string(argv[1]) == "--fuzz") {
    fuzz(atoi(argv[2]));
    printf("tiles of the forward kernel served by the INNER ('reflection', inside the image) copy of the unit code: %lld of %lld\n", emu_inner_tiles,
           emu_inner_tiles + emu_other_tiles);
    printf("%s: %d failing comparisons in the fuzz run\n", failures ? "FAILED" : "PASSED", failures);
    return failures ? 1 : 0;
  }
  test_u8_all();
  for (int lazy = 0; lazy < 2; ++lazy) {
    // grids that do not divide the number of strips / bands: segments that start in the middle of a band
    test_sepfilter<11, KB200_REFLECT>(2, 3, 70, 132, 5, lazy);
    test_sepfilter<11, KB200_REPLICATE>(1, 2, 97, 260, 4, lazy);
    test_sepfilter<11, KB200_CONSTANT>(1, 1, 33, 4, 1, lazy);
    test_sepfilter<3, KB200_REFLECT>(2, 1, 32, 128, 2, lazy);
    test_sepfilter<5, KB200_REPLICATE>(1, 1, 6, 8, 1, lazy);
    test_sepfilter<17, KB200_REFLECT>(1, 2, 130, 140, 3, lazy);
    test_sepfilter<17, KB200_CONSTANT>(1, 1, 64, 388, 7, lazy);
    test_pyrdown<KB200_REFLECT>(3, 70, 132, 4, lazy);
    test_pyrdown<KB200_REPLICATE>(2, 34, 260, 3, lazy);
    test_pyrdown<KB200_CONSTANT>(1, 4, 4, 1, lazy);
    test_gradient<3, 2, false>(3, 70, 132, 4, lazy);
    test_gradient<3, 2, true>(2, 33, 260, 3, lazy);
    test_gradient<3, 3, false>(1, 3, 4, 1, lazy);
    test_gradient<5, 3, false>(2, 97, 136, 5, lazy);
    test_ssim<11>(3, 70, 132, 4, lazy);
    test_ssim<5>(2, 33, 8, 1, lazy);
    test_ssim<3>(1, 32, 64, 1, lazy);
    test_ssim<7>(2, 97, 260, 7, lazy);
    test_ssim<9>(1, 6, 8, 1, lazy);
    if (!lazy) test_reflect_near();
    test_undistort(2, 70, 132, lazy);
    test_undistort(1, 33, 64, lazy);
    test_undistort(2, 97, 200, lazy, true);
    test_forward<true, KB200_ZEROS, 64, 32, 72, 40>(3, 96, 200, 96, 200, 3, lazy, true);
    test_forward<true, KB200_ZEROS, 64, 32, 72, 40>(3, 70, 132, 50, 100, 2, lazy, false);
    test_forward<false, KB200_BORDER, 64, 32, 72, 40>(3, 64, 128, 70, 132, 4, lazy, true);
    test_forward<true, KB200_ZEROS, 32, 32, 56, 56>(3, 70, 132, 70, 132, 3, lazy, false);
    test_forward<true, KB200_REFLECTION, 64, 32, 72, 40>(3, 70, 132, 70, 132, 3, lazy, false);
    test_forward<true, KB200_FILL, 64, 32, 72, 40>(3, 70, 132, 64, 120, 2, lazy, true);
    test_forward<true, KB200_ZEROS, 64, 32, 72, 40, KB200_NEAREST>(3, 70, 132, 70, 132, 3, lazy, true);
    test_forward<true, KB200_BORDER, 64, 32, 72, 40, KB200_BICUBIC>(3, 70, 132, 70, 132, 2, lazy, true);
    test_forward<false, KB200_REFLECTION, 64, 32, 72, 40, KB200_BICUBIC>(3, 64, 128, 70, 132, 3, lazy, false);
    test_backward<true>(3, 70, 132, 70, 132, 2, lazy);
    test_backward<false>(3, 64, 128, 50, 96, 3, lazy);
    test_backward<true>(3, 40, 72, 66, 132, 4, lazy);
    test_backward<true>(3, 96, 200, 96, 200, 3, lazy, true);
    test_backward<false>(2, 70, 132, 70, 132, 5, lazy, true);
  }
  printf("%s: %d failing comparisons, %lld TMA loads, %lld TMA reduce-adds, %lld CTA barriers and %lld warp rendezvous emulated\n",
         failures ? "FAILED" : "PASSED", failures, emu::n_tma, emu::n_reduce, emu::n_barriers, emu::n_wsync);
  return failures ? 1 : 0;
}
