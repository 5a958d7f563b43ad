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
#include "../../kornia_b200/csrc/filter2d_taps.cuh"
#include "../../kornia_b200/csrc/gradient_tiled.cuh"
#include "../../kornia_b200/csrc/ssim_vwalk.cuh"
#include "../../kornia_b200/csrc/corner_vwalk.cuh"
#include "../../kornia_b200/csrc/octave_vwalk.cuh"
#include "../../kornia_b200/csrc/nms.cuh"
#include "../../kornia_b200/csrc/quad_interp.cuh"
#include "../../kornia_b200/csrc/siftdesc.cuh"
#include "../../kornia_b200/csrc/patch_orientation.cuh"
#include "../../kornia_b200/csrc/laf_patches.cuh"
#include "../../kornia_b200/csrc/affine_shape.cuh"
#include "../../kornia_b200/csrc/remap_tiled.cuh"
#include "ref_ssim_tiled.cuh"
#include "../../kornia_b200/csrc/warp_bwd_tma2.cuh"
#include "../../kornia_b200/csrc/warp_u8_tiled.cuh"

#include <random>
#include <string>

namespace kb200 {
alignas(128) unsigned char sept_smem[256 * 1024];
alignas(128) unsigned char f2d_smem[256 * 1024];
alignas(128) unsigned char f2dt_smem[128 * 1024];
alignas(128) unsigned char nms_smem[64 * 1024];
alignas(128) unsigned char gradt_smem[256 * 1024];
alignas(128) unsigned char ssimv_smem[256 * 1024];
alignas(128) unsigned char corner_smem[256 * 1024];
alignas(128) unsigned char oct_smem[256 * 1024];
alignas(128) float ssim_smem[64 * 1024];
alignas(128) unsigned char remap_smem[256 * 1024];
alignas(128) unsigned char tma_smem[256 * 1024];
alignas(128) unsigned char bwd2_smem[256 * 1024];
alignas(128) unsigned char u8t_smem[256 * 1024];
alignas(128) unsigned char sift_smem[128 * 1024];
alignas(128) unsigned char ori_smem[128 * 1024];
alignas(128) unsigned char paff_smem[64 * 1024];
alignas(128) unsigned char laff_smem[64 * 1024];
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
// bit for bit, -0 != +0: every case of the fixed list and of the fuzz run holds to it (a kernel that seeded an accumulator
// or folded a border differently from the scalar loop would show as a zero of the other sign)
static void compare(const std::string& what, const float* got, const float* want, size_t n) {
  size_t bad = 0, first = 0;
  for (size_t i = 0; i < n; ++i)
    if (memcmp(got + i, want + i, 4) != 0) {
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

static int emu_strict_failures = 0;
// bits equal (-0 != +0), or NaN on both sides: the device returns one canonical NaN, while on x86 the sign of a NaN produced
// from two NaN operands depends on which operand the compiler put first in a commutative op
static void compare_bits_or_nan(const std::string& what, const float* got, const float* want, size_t n) {
  size_t bad = 0, first = 0;
  for (size_t i = 0; i < n; ++i)
    if (memcmp(got + i, want + i, 4) != 0 && !(got[i] != got[i] && want[i] != want[i])) {
      if (!bad) first = i;
      ++bad;
    }
  if (bad) {
    printf("FAIL %-72s %zu / %zu differ in their bits, first at %zu: got %.9g want %.9g\n", what.c_str(), bad, n, first, got[first], want[first]);
    ++failures;
    ++emu_strict_failures;
  } else {
    printf("ok   %s\n", what.c_str());
  }
}

// specials 1: NaN / +-Inf / -0 / subnormal / 1e-38 / 3e38 texels scattered; 2: the same, and the first plane all -0 (a
// kernel that seeds an accumulator differently from the scalar loop shows there as +0 against -0).
static void special_texels(float* x, size_t n, int specials, size_t plane = 0) {
  if (!specials) return;
  const float v[8] = {NAN, INFINITY, -INFINITY, -0.f, 1e-40f, -1e-41f, 1e-38f, 3e38f};
  for (size_t i = 0; i < n; i += 97 + (rng() % 300)) x[i] = v[rng() % 8];
  x[0] = 1e-40f;
  x[n - 1] = -0.f;
  if (specials >= 2 && plane && plane < n)
    for (size_t i = 0; i < plane; ++i) x[i] = -0.f;
}

// the comparison of a case: with special texels bit for bit (-0 != +0, any NaN equals any NaN)
static void compare_case(int specials, const std::string& what, const float* got, const float* want, size_t n) {
  if (specials) compare_bits_or_nan(what + " specials=" + std::to_string(specials), got, want, n);
  else compare(what, got, want, n);
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
static void test_sepfilter(int B, int C, int H, int W, unsigned grid, bool lazy, int specials = 0) {
  emu::lazy_tma = lazy;
  const int planes = B * C;
  std::vector<float> xs, o1s, o2s;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  special_texels(x, (size_t)planes * H * W, specials, (size_t)H * W);
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
    compare_case(specials, "sepfilter_tiled_kernel (verified on hw) " + tag, o1, want.data(), want.size());
  }
  if (K <= 11) {  // unsharp_mask epilogue against the plain filter blended on the host (|w| < 0.5 and >= 0.5 take different forms)
    const float wts[2] = {0.3f, 2.0f};
    const float wt = wts[(H + W) & 1];
    std::vector<float> blended(want.size());
    for (size_t i = 0; i < want.size(); ++i) blended[i] = lerp_like_torch(o1[i], x[i], wt);
    const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
    SepTiledParams p{kx.data(), ky.data(), o2, C, H, W, B, 1, planes, x, wt};
    emu::launch(grid, dim3(256), [&] { sepfilter_tiled_kernel<K, BORDER, true>(map, p); });
    compare_case(specials, "sepfilter_tiled_kernel<LERP> vs lerp of the plain filter " + tag, o2, blended.data(), want.size());
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
static void test_pyrdown(int planes, int H, int W, unsigned grid, bool lazy, int specials = 0) {
  emu::lazy_tma = lazy;
  std::vector<float> xs, os, fs;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  special_texels(x, (size_t)planes * H * W, specials, (size_t)H * W);
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
    compare_case(specials, "filter2d_tiled_kernel<5> (verified on hw) " + tag, o, full.data(), full.size());
  }
  {
    float* o = aligned(os, want.size());
    F2dTiledParams p{taps, o, 1, H, W, 1, planes};
    emu::launch(grid, dim3(256), [&] { filter2d_tiled_kernel<5, BORDER, true>(map, p); });
    compare_case(specials, "filter2d_tiled_kernel<5, DOWN2> (pyrdown)  " + tag, o, want.data(), want.size());
  }
}

template <int K, int BORDER>
static void test_filter2d(int planes, int H, int W, unsigned grid, bool lazy, int specials = 0) {
  emu::lazy_tma = lazy;
  std::vector<float> xs, os;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  special_texels(x, (size_t)planes * H * W, specials, (size_t)H * W);
  auto taps = randv(K * K, -1.f, 1.f);
  std::vector<float> want((size_t)planes * H * W);
  ref_filter2d(x, taps.data(), 1, want.data(), planes, H, W, K, BORDER);
  float* o = aligned(os, want.size());
  const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
  F2dTiledParams p{taps.data(), o, 1, H, W, 1, planes};
  emu::launch(grid, dim3(256), [&] { filter2d_tiled_kernel<K, BORDER, false>(map, p); });
  compare_case(specials, "filter2d_tiled_kernel (verified on hw) K=" + std::to_string(K) + " border=" + std::to_string(BORDER) + " " + std::to_string(planes) + "x" +
              std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"),
          o, want.data(), want.size());
}

// ------------------------------------------------------------------------------------------ filter2d, zero-skipping (K 9..31)
static void compare_bits(const std::string& what, const float* got, const float* want, size_t n) {  // -0 != +0 here
  size_t bad = 0, first = 0;
  for (size_t i = 0; i < n; ++i)
    if (memcmp(got + i, want + i, 4) != 0) {
      if (!bad) first = i;
      ++bad;
    }
  if (bad) {
    printf("FAIL %-72s %zu / %zu differ in their bits, first at %zu: got %.9g want %.9g\n", what.c_str(), bad, n, first, got[first], want[first]);
    ++failures;
    ++emu_strict_failures;
  } else {
    printf("ok   %s\n", what.c_str());
  }
}

// kind 0: a nearest-rotated line (K .. 1.4 K taps), 1: a bilinear-rotated line (~3 K taps), 2: dense, 3: a line with
// subnormal weights, 4: no nonzero tap at all.  Zero taps are a mix of +0 and -0.
static void make_taps(float* k, int K, int kind) {
  std::uniform_real_distribution<float> u(0.05f, 1.f);
  for (int t = 0; t < K * K; ++t) k[t] = (rng() & 1) ? 0.f : -0.f;
  if (kind == 4) return;
  if (kind == 2) {
    for (int t = 0; t < K * K; ++t) k[t] = u(rng) - 0.5f;
    return;
  }
  const float a = std::uniform_real_distribution<float>(0.f, 3.14159265f)(rng);
  const float c = (K - 1) * 0.5f, dx = cosf(a), dy = sinf(a);
  for (int s = 0; s < 4 * K; ++s) {
    const float r = -c + (2.f * c) * s / (4 * K - 1);
    const float fx = c + r * dx, fy = c + r * dy;
    if (kind == 1) {
      const int x0 = (int)floorf(fx), y0 = (int)floorf(fy);
      for (int dyy = 0; dyy < 2; ++dyy)
        for (int dxx = 0; dxx < 2; ++dxx)
          if (x0 + dxx < K && y0 + dyy < K) k[(y0 + dyy) * K + x0 + dxx] = u(rng) / K;
    } else {
      k[(int)lrintf(fy) * K + (int)lrintf(fx)] = kind == 3 ? 1e-41f : u(rng) / K;
    }
  }
}

// specials: 0 none; 1 NaN / +-Inf / -0 / subnormal texels in a few places; 2 tiny texels whose products with the taps
// underflow (the case where a skipped fma(0, v, -0) would show); 3 every texel -0.
template <int BORDER>
static void test_taps(int K, int B, int C, int H, int W, int Bk, int kind, int specials, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  const int planes = B * C;
  std::vector<float> xs, os, ks((size_t)Bk * K * K);
  float* x = aligned(xs, (size_t)planes * H * W);
  std::uniform_real_distribution<float> u(-1.f, 1.f);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = specials == 3 ? -0.f : specials == 2 ? u(rng) * 1e-30f : u(rng);
  if (specials == 1) {
    const float sp[6] = {NAN, INFINITY, -INFINITY, -0.f, 1e-40f, -3e-39f};
    for (int s = 0; s < 12; ++s) x[(size_t)(rng() % ((size_t)planes * H * W))] = sp[s % 6];
  }
  for (int b = 0; b < Bk; ++b) make_taps(ks.data() + (size_t)b * K * K, K, kind == 5 ? b % 5 : kind);
  std::vector<float> want((size_t)planes * H * W);
  const int h = (K - 1) / 2;
  for (int pl = 0; pl < planes; ++pl) {
    const float* kp = ks.data() + (size_t)((pl / C) % Bk) * K * K;
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        float a = 0.f;
        for (int i = 0; i < K; ++i)
          for (int j = 0; j < K; ++j) {
            const int sy = fold(y + i - h, H, BORDER), sx = fold(xx + j - h, W, BORDER);
            a = fmaf(kp[i * K + j], (sy < 0 || sx < 0) ? 0.f : x[(size_t)pl * H * W + (size_t)sy * W + sx], a);
          }
        want[((size_t)pl * H + y) * W + xx] = a;
      }
  }
  float* o = aligned(os, want.size());
  for (size_t i = 0; i < want.size(); ++i) o[i] = NAN;
  const CUtensorMap map = emu::make_map(x, W, H, planes, F2DT_BW, SEPT_TH + K - 1, 1);
  F2dTapsParams p{ks.data(), o, C, H, W, Bk, planes, K};
  emu::set_smem(f2dt_smem, sizeof(f2dt_smem));
  if (f2d_taps_smem_bytes(K) > sizeof(f2dt_smem)) emu::fail("filter2d_taps_kernel: shared memory of the CTA exceeds the emulated array");
  emu::launch(grid, dim3(256), [&] { filter2d_taps_kernel<BORDER>(map, p); });
  compare_bits("filter2d_taps_kernel vs the dense loop K=" + std::to_string(K) + " border=" + std::to_string(BORDER) + " " + std::to_string(B) + "x" +
                   std::to_string(C) + "x" + std::to_string(H) + "x" + std::to_string(W) + " Bk=" + std::to_string(Bk) + " kind=" + std::to_string(kind) +
                   " specials=" + std::to_string(specials) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"),
               o, want.data(), want.size());
}

// The fixed list (also alone: run_emu --taps).  Kernel kinds 0 nearest line, 1 bilinear line, 2 dense, 3 subnormal taps,
// 4 all zero, 5 one of each per sample; Bk 1, B and cycling; grids that do not divide the strips; special texels.
static void test_taps_all(bool lazy) {
  test_taps<KB200_CONSTANT>(9, 2, 3, 70, 132, 2, 0, 0, 5, lazy);
  test_taps<KB200_REFLECT>(15, 3, 1, 97, 260, 1, 1, 1, 4, lazy);
  test_taps<KB200_REPLICATE>(31, 3, 2, 40, 136, 2, 5, 1, 3, lazy);
  test_taps<KB200_REFLECT>(31, 1, 1, 16, 20, 1, 2, 2, 1, lazy);
  test_taps<KB200_CONSTANT>(15, 2, 1, 33, 8, 2, 3, 0, 2, lazy);
  test_taps<KB200_REPLICATE>(9, 1, 2, 35, 64, 1, 4, 3, 2, lazy);
  test_taps<KB200_CONSTANT>(21, 4, 1, 50, 100, 3, 5, 2, 3, lazy);
  test_taps<KB200_REFLECT>(9, 5, 1, 64, 256, 5, 0, 1, 7, lazy);
  test_taps<KB200_REFLECT>(15, 2, 1, 40, 64, 2, 3, 2, 3, lazy);  // products that underflow: acc = -0 before a zero tap
}

template <int K, int NOUT, bool MAG>
static void test_gradient(int planes, int H, int W, unsigned grid, bool lazy, int specials = 0) {
  emu::lazy_tma = lazy;
  std::vector<float> xs, os;
  float* x = aligned(xs, (size_t)planes * H * W);
  for (size_t i = 0; i < (size_t)planes * H * W; ++i) x[i] = randv(1)[0];
  special_texels(x, (size_t)planes * H * W, specials, (size_t)H * W);
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
  emu::launch(grid, dim3(256), [&] { grad_tiled_kernel<K, NOUT, MAG ? GRAD_MAG : GRAD_PLANES>(map, p); });
  compare_case(specials, "grad_tiled_kernel K=" + std::to_string(K) + " NOUT=" + std::to_string(NOUT) + (MAG ? " MAG " : "     ") + std::to_string(planes) + "x" +
              std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"),
          p.out, want.data(), want.size());
}

// ------------------------------------------------------------------------------------------ SSIM
template <int K>
static void test_ssim(int planes, int H, int W, unsigned grid, bool lazy, int specials = 0) {
  emu::lazy_tma = lazy;
  std::vector<float> as, bs, o1s, o2s;
  const size_t n = (size_t)planes * H * W;
  float* a = aligned(as, n);
  float* b = aligned(bs, n);
  for (size_t i = 0; i < n; ++i) {
    a[i] = randv(1)[0];
    b[i] = std::min(1.f, std::max(0.f, a[i] + randv(1, -0.1f, 0.1f)[0]));
  }
  special_texels(a, n, specials, (size_t)H * W);
  special_texels(b, n, specials ? 1 : 0);
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
    const CUtensorMap ma = emu::make_map(a, W, H, planes, VWALK_BW, VWALK_TH, 1), mb = emu::make_map(b, W, H, planes, VWALK_BW, VWALK_TH, 1);
    const CUtensorMap pa = emu::make_map(a, W, H, planes, VWALK_BW, K - 1, 1), pb = emu::make_map(b, W, H, planes, VWALK_BW, K - 1, 1);
    SsimVParams p{taps.data(), o2, planes, H, W, C1, C2, eps};
    emu::launch(grid, dim3(256), [&] { ssim_vwalk_kernel<K>(ma, mb, pa, pb, p); });
  }
  compare_case(specials, "ssim_vwalk_kernel vs ssim_tiled_kernel " + tag, o2, o1, n);
}


// ------------------------------------------------------------------------------------------ ScalePyramid octave
// Scalar restatement of one octave as this library composes it: level 0 the source or its filter2d_separable with the
// initial taps, level l the filter2d_separable of level l-1 (row pass, then column pass, ascending FMA from 0, reflect
// border of the level it filters).  Compared bit for bit (-0 != +0, NaN equals NaN) with octave_vwalk_kernel, whose
// output is prefilled with a value no level produces.
template <typename CH>
static void test_octave(int planes, int H, int W, int specials, unsigned grid) {
  constexpr int L = CH::L;
  const size_t HW = (size_t)H * W, n = (size_t)planes * HW;
  std::vector<float> xs, os;
  float* x = aligned(xs, n);
  for (size_t i = 0; i < n; ++i) x[i] = randv(1, -1.f, 2.f)[0];
  special_texels(x, n, specials, HW);
  OctaveParams p{};
  for (int l = 0; l < L; ++l) {
    const int K = CH::K[l];
    float s = 0.f;
    const float sig = 0.15f * K + 0.1f * (float)l;
    for (int j = 0; j < K; ++j) s += (p.taps[l][j] = expf(-0.5f * (float)((j - K / 2) * (j - K / 2)) / (sig * sig)));
    for (int j = 0; j < K; ++j) p.taps[l][j] /= s;
  }
  std::vector<float> want(n * L), row(HW);
  for (int pl = 0; pl < planes; ++pl) {
    for (int l = 0; l < L; ++l) {
      float* dst = want.data() + ((size_t)pl * L + l) * HW;
      const float* prev = l == 0 ? x + pl * HW : dst - HW;
      if (l == 0 && !CH::BLUR0) {
        std::copy(prev, prev + HW, dst);
        continue;
      }
      const int K = CH::K[l], h = K / 2;
      for (int y = 0; y < H; ++y)
        for (int xx = 0; xx < W; ++xx) {
          float a = 0.f;
          for (int j = 0; j < K; ++j) a = fmaf(p.taps[l][j], prev[(size_t)y * W + fold(xx + j - h, W, KB200_REFLECT)], a);
          row[y * W + xx] = a;
        }
      for (int y = 0; y < H; ++y)
        for (int xx = 0; xx < W; ++xx) {
          float a = 0.f;
          for (int i = 0; i < K; ++i) a = fmaf(p.taps[l][i], row[(size_t)fold(y + i - h, H, KB200_REFLECT) * W + xx], a);
          dst[(size_t)y * W + xx] = a;
        }
    }
  }
  float* out = aligned(os, n * L);
  std::fill(out, out + n * L, -777.f);
  p.src = x;
  p.out = out;
  p.planes = planes;
  p.H = H;
  p.W = W;
  emu::launch(grid, dim3(OCT_NT), [&] { octave_vwalk_kernel<CH>(p); });
  std::string chain = std::to_string(CH::K[0] * CH::BLUR0);
  for (int l = 1; l < L; ++l) chain += "," + std::to_string(CH::K[l]);
  compare_bits_or_nan("octave_vwalk_kernel [" + chain + "] " + std::to_string(planes) + "x" + std::to_string(H) + "x" + std::to_string(W) +
                          (specials ? " special texels" : "") + " grid=" + std::to_string(grid),
                      out, want.data(), n * L);
}

using OctDefault = OctaveChain<13, 11, 13, 17, 21, 25>;
using OctDetector = OctaveChain<13, 11, 13, 17, 21>;
using OctDouble = OctaveChain<11, 11, 13, 17, 21, 25>;
using OctCopy6 = OctaveChain<0, 11, 13, 17, 21, 25>;
using OctCopy5 = OctaveChain<0, 11, 13, 17, 21>;

// One octave of a chain on a shape and grid, with finite and special texels.
template <typename CH>
static void test_octave_both(int planes, int H, int W, unsigned grid) {
  test_octave<CH>(planes, H, W, 0, grid);
  test_octave<CH>(planes, H, W, 2, grid);
}

// The fixed list (also alone: run_emu --octave): every instantiation in both stage-0 modes; the smallest side equal to the
// largest tap count (25 x 28, 21 x 60 for the 21-tap chains); widths 28, 60, 132 (a band of 4 columns); heights that are
// not a multiple of the 16-row step; grids larger than the number of bands (segments that start in the middle of a band,
// after the priming steps) and grids that do not divide them.
static void test_octave_all() {
  test_octave_both<OctDefault>(2, 25, 28, 1);
  test_octave_both<OctDefault>(1, 70, 132, 3);
  test_octave_both<OctDefault>(2, 97, 60, 7);
  test_octave_both<OctDetector>(1, 21, 60, 2);
  test_octave_both<OctDetector>(2, 61, 132, 5);
  test_octave_both<OctDouble>(1, 33, 260, 4);
  test_octave_both<OctDouble>(3, 26, 28, 2);
  test_octave_both<OctCopy6>(1, 25, 132, 2);
  test_octave_both<OctCopy6>(2, 83, 60, 9);
  test_octave_both<OctCopy5>(1, 21, 28, 1);
  test_octave_both<OctCopy5>(2, 140, 68, 11);
}

// ------------------------------------------------------------------------------------------ non-maximum suppression
// Scalar restatement of kornia/geometry/subpix/nms.py: a position is kept when it is strictly greater than every
// neighbour (explicit K = 3, 5, 7: in-image neighbours, the (K - 1) / 2 ring False; K >= 9: replicate-clamped neighbours
// and 0, and False when the window holds a non-finite texel), in 3-D than its 26 neighbours (strictly smaller for the
// minima), the border levels, rows and columns False.  Values are x * keep.  The source planes sit at a plane stride that
// is not H * W (a permuted view), and texels are quantised to quarters so ties are common.
static void nms_source(std::vector<float>& store, float*& x, size_t planes, size_t stride, size_t HW, int specials) {
  x = aligned(store, planes * stride);
  for (size_t i = 0; i < planes * stride; ++i) x[i] = (float)(rng() % 7) * 0.25f - 0.75f;
  if (specials)
    for (size_t p = 0; p < planes; ++p) special_texels(x + p * stride, HW, 1);
}

static void nms_bytes_as_float(const std::vector<unsigned char>& m, std::vector<float>& f) {
  f.resize(m.size());
  for (size_t i = 0; i < m.size(); ++i) f[i] = (float)m[i];
}

template <int K, bool VALUES>
static void test_nms2d(int B, int C, int H, int W, int specials, unsigned grid) {
  constexpr int R = K / 2;
  const size_t HW = (size_t)H * W, planes = (size_t)B * C, stride = HW + 5;
  std::vector<float> xs;
  float* x;
  nms_source(xs, x, planes, stride, HW, specials);
  std::vector<float> want(planes * HW), got(planes * HW);
  for (size_t pl = 0; pl < planes; ++pl)
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        const float* src = x + pl * stride;
        const float c = src[(size_t)y * W + xx];
        bool keep = K > 7 ? (bool)std::isfinite(c) && c > 0.f : y >= R && y < H - R && xx >= R && xx < W - R;
        for (int dy = -R; dy <= R && keep; ++dy)
          for (int dx = -R; dx <= R && keep; ++dx) {
            const float n = src[(size_t)fold(y + dy, H, KB200_REPLICATE) * W + fold(xx + dx, W, KB200_REPLICATE)];
            if (K > 7 && !std::isfinite(n)) keep = false;
            else if ((dy || dx) && !(c > n)) keep = false;
          }
        want[pl * HW + (size_t)y * W + xx] = VALUES ? c * (keep ? 1.f : 0.f) : (float)keep;
      }
  Nms2dParams p{};
  p.src = x;
  p.sB = (long long)C * stride;
  p.sC = (long long)stride;
  p.C = C;
  p.H = H;
  p.W = W;
  p.tiles_x = ceil_div(W, NMS_TW);
  p.tiles_y = ceil_div(H, NMS_TH);
  p.tiles = (long long)planes * p.tiles_x * p.tiles_y;
  std::vector<float> os;
  std::vector<unsigned char> om(planes * HW + 16, 0xff);
  if (VALUES) {
    p.out = aligned(os, planes * HW);
  } else {
    p.out = om.data();
  }
  emu::launch(grid, dim3(NMS_NT), [&] { nms2d_kernel<K, VALUES>(p); });
  if (VALUES) std::copy((float*)p.out, (float*)p.out + planes * HW, got.begin());
  else nms_bytes_as_float(std::vector<unsigned char>(om.begin(), om.begin() + planes * HW), got);
  compare_bits_or_nan("nms2d_kernel K=" + std::to_string(K) + (VALUES ? " values " : " mask ") + std::to_string(B) + "x" + std::to_string(C) + "x" +
                          std::to_string(H) + "x" + std::to_string(W) + (specials ? " special texels" : "") + " grid=" + std::to_string(grid),
                      got.data(), want.data(), planes * HW);
}

template <int MODE>
static void test_nms3d(int B, int C, int L, int H, int W, int specials, unsigned grid) {
  const size_t HW = (size_t)H * W, vols = (size_t)B * C, lstride = HW + 3, n = vols * L * HW;
  std::vector<float> xs;
  float* x;
  nms_source(xs, x, vols * L, lstride, HW, specials);
  // (B, L, C, H, W) storage read as (B, C, L, H, W): the permuted view ScaleSpaceDetector hands over
  const long long sC = (long long)lstride, sL = (long long)C * lstride, sB = (long long)L * C * lstride;
  std::vector<float> wmax(n), wmin(n), got(n);
  for (size_t v = 0; v < vols; ++v) {
    const float* src = x + (v / C) * sB + (v % C) * sC;
    for (int l = 0; l < L; ++l)
      for (int y = 0; y < H; ++y)
        for (int xx = 0; xx < W; ++xx) {
          const float c = src[l * sL + (size_t)y * W + xx];
          bool kmax = l >= 1 && l < L - 1 && y >= 1 && y < H - 1 && xx >= 1 && xx < W - 1, kmin = kmax;
          for (int dl = -1; dl <= 1 && (kmax || kmin); ++dl)
            for (int dy = -1; dy <= 1; ++dy)
              for (int dx = -1; dx <= 1; ++dx) {
                if (!dl && !dy && !dx) continue;
                const float nb = src[(l + dl) * sL + (size_t)(y + dy) * W + xx + dx];
                kmax = kmax && c > nb;
                kmin = kmin && c < nb;
              }
          const size_t o = ((v * L + l) * H + y) * W + xx;
          wmax[o] = MODE == NMS3_MAX_VALUES ? c * (kmax ? 1.f : 0.f) : (float)kmax;
          wmin[o] = (float)kmin;
        }
  }
  Nms3dParams p{};
  p.src = x;
  p.sB = sB;
  p.sC = sC;
  p.sL = sL;
  p.C = C;
  p.L = L;
  p.H = H;
  p.W = W;
  p.tiles_x = ceil_div(W, NMS3_TW);
  p.tiles_y = ceil_div(H, NMS3_TH);
  p.tiles = (long long)vols * p.tiles_x * p.tiles_y;
  std::vector<float> os;
  std::vector<unsigned char> o0(n, 0xff), o1(n, 0xff);
  p.out0 = MODE == NMS3_MAX_VALUES ? (void*)aligned(os, n) : (void*)o0.data();
  p.out1 = o1.data();
  emu::launch(grid, dim3(NMS3_NT), [&] { nms3d_kernel<MODE>(p); });
  const std::string what = std::string("nms3d_kernel ") + (MODE == NMS3_MAX_MASK ? "mask " : MODE == NMS3_MAX_VALUES ? "values " : "minmax ") +
                           std::to_string(B) + "x" + std::to_string(C) + "x" + std::to_string(L) + "x" + std::to_string(H) + "x" + std::to_string(W) +
                           (specials ? " special texels" : "") + " grid=" + std::to_string(grid);
  if (MODE == NMS3_MAX_VALUES) std::copy((float*)p.out0, (float*)p.out0 + n, got.begin());
  else nms_bytes_as_float(o0, got);
  compare_bits_or_nan(what + (MODE == NMS3_MINMAX ? " (maxima)" : ""), got.data(), wmax.data(), n);
  if (MODE == NMS3_MINMAX) {
    nms_bytes_as_float(o1, got);
    compare_bits_or_nan(what + " (minima)", got.data(), wmin.data(), n);
  }
}

template <int K>
static void test_nms2d_both(int B, int C, int H, int W, int specials, unsigned grid) {
  test_nms2d<K, false>(B, C, H, W, specials, grid);
  test_nms2d<K, true>(B, C, H, W, specials, grid);
}

// The fixed list (also alone: run_emu --nms): every instantiated K in both forms on a shape with partial edge tiles;
// tiles that lie wholly inside the halo (H or W below K, 1 x 1, 2 x 2); grids that do not divide the tiles; and the 3-D
// kernel in all three modes on odd widths, level counts 1, 2, 3 and 5, with finite and special texels.
static void test_nms_all() {
  test_nms2d_both<3>(1, 2, 70, 131, 1, 5);
  test_nms2d_both<5>(2, 1, 33, 67, 0, 3);
  test_nms2d_both<7>(1, 1, 40, 130, 1, 2);
  test_nms2d_both<9>(1, 2, 45, 70, 1, 4);
  test_nms2d_both<11>(1, 1, 33, 65, 0, 1);
  test_nms2d_both<13>(1, 1, 36, 66, 1, 2);
  test_nms2d_both<15>(2, 1, 61, 68, 1, 3);
  test_nms2d_both<17>(1, 1, 20, 70, 0, 2);
  test_nms2d_both<19>(1, 1, 34, 40, 1, 1);
  test_nms2d_both<21>(1, 1, 30, 15, 1, 2);
  test_nms2d_both<23>(1, 1, 40, 65, 0, 2);
  test_nms2d_both<25>(1, 1, 33, 30, 1, 1);
  test_nms2d_both<27>(1, 1, 26, 80, 0, 2);
  test_nms2d_both<29>(1, 1, 35, 66, 1, 2);
  test_nms2d_both<31>(1, 2, 40, 70, 1, 3);
  test_nms2d_both<7>(1, 1, 5, 3, 1, 1);
  test_nms2d_both<15>(1, 1, 9, 6, 1, 1);
  test_nms2d_both<3>(2, 1, 1, 1, 0, 1);
  test_nms2d_both<9>(1, 1, 1, 1, 1, 1);
  test_nms2d_both<5>(1, 1, 2, 2, 0, 1);
  test_nms2d_both<31>(1, 1, 2, 2, 1, 1);
  for (int sp = 0; sp < 2; ++sp) {
    test_nms3d<NMS3_MINMAX>(1, 2, 5, 19, 131, sp, 3);
    test_nms3d<NMS3_MAX_MASK>(2, 1, 3, 9, 30, sp, 2);
    test_nms3d<NMS3_MAX_VALUES>(1, 1, 4, 17, 15, sp, 1);
    test_nms3d<NMS3_MINMAX>(1, 1, 2, 5, 5, sp, 1);
    test_nms3d<NMS3_MINMAX>(1, 1, 1, 1, 1, sp, 1);
    test_nms3d<NMS3_MAX_VALUES>(1, 2, 3, 3, 3, sp, 2);
  }
}

// ------------------------------------------------------------------------------------------ sub-pixel refinement
// Scalar restatement of conv_quad_interp3d / iterative_quad_interp3d (kornia/geometry/subpix/spatial_soft_argmax.py):
// every maximum (the given mask, or strictly above its 26 neighbours with the border False) runs all n_iters iterations
// (a failed keypoint is frozen), solving the 3 x 3 x 3 fit at its clamped position in the reference's operation order;
// the conv form also needs a mask voxel within L-inf `radius`.  The source is a permuted (B, L, C, H, W) store read as
// (B, C, L, H, W), texels are normal draws (keypoints walk) or special values.
static void test_quad(int B, int C, int L, int H, int W, int radius, bool has_mask, int n_iters, float shift, float bonus, bool allow,
                      int specials, unsigned grid) {
  const size_t HW = (size_t)H * W, vols = (size_t)B * C, lstride = HW + 3, n = vols * L * HW;
  std::vector<float> xs;
  float* x = aligned(xs, vols * L * lstride);
  std::normal_distribution<float> nd(0.f, 1.f);
  for (size_t i = 0; i < vols * L * lstride; ++i) x[i] = nd(rng);
  if (specials)
    for (size_t p = 0; p < vols * L; ++p) special_texels(x + p * lstride, HW, 1);
  const long long sC = (long long)lstride, sL = (long long)C * lstride, sB = (long long)L * C * lstride;
  std::vector<unsigned char> mask(n, 0);
  for (size_t i = 0; i < n; ++i) mask[i] = rng() % 25 == 0 || (i / W) % H == 0;  // sparse, and every first row
  auto src = [&](size_t v, int d, int h, int w) { return x[(v / C) * sB + (v % C) * sC + d * sL + (size_t)h * W + w]; };
  auto is_max = [&](size_t v, int d, int h, int w) {
    if (has_mask) return mask[((v * L + d) * H + h) * W + w] != 0;
    if (d < 1 || d > L - 2 || h < 1 || h > H - 2 || w < 1 || w > W - 2) return false;
    const float c = src(v, d, h, w);
    bool k = true;
    for (int a = -1; a <= 1; ++a)
      for (int b = -1; b <= 1; ++b)
        for (int e = -1; e <= 1; ++e)
          if ((a || b || e) && !(c > src(v, d + a, h + b, w + e))) k = false;
    return k;
  };
  std::vector<float> wc(3 * n), wy(n);
  const bool refine = L >= 3 && H >= 3 && W >= 3;
  for (size_t v = 0; v < vols; ++v)
    for (int d0 = 0; d0 < L; ++d0)
      for (int h0 = 0; h0 < H; ++h0)
        for (int w0 = 0; w0 < W; ++w0) {
          const size_t o = ((v * L + d0) * H + h0) * W + w0, co = ((v * 3 * L + d0) * H + h0) * W + w0;
          float cs = (float)d0, cx = (float)w0, cy = (float)h0, y = src(v, d0, h0, w0);
          if (refine && is_max(v, d0, h0, w0)) {
            int d = d0, h = h0, w = w0;
            bool valid = true;
            float s[3] = {0.f, 0.f, 0.f}, gds = 0.f;  // x, y, level
            for (int it = 0; it < n_iters; ++it) {
              if (!valid) continue;
              const int dc = std::min(std::max(d, 1), L - 2), hc = std::min(std::max(h, 1), H - 2), wc_ = std::min(std::max(w, 1), W - 2);
              auto P = [&](int a, int b, int e) { return src(v, dc + a, hc + b, wc_ + e); };
              const float g[3] = {0.5f * (P(0, 0, 1) - P(0, 0, -1)), 0.5f * (P(0, 1, 0) - P(0, -1, 0)), 0.5f * (P(1, 0, 0) - P(-1, 0, 0))};
              const float c2 = 2.f * P(0, 0, 0);
              const float dxx = P(0, 0, 1) - c2 + P(0, 0, -1), dyy = P(0, 1, 0) - c2 + P(0, -1, 0), dss = P(1, 0, 0) - c2 + P(-1, 0, 0);
              const float dxy = 0.25f * (P(0, 1, 1) - P(0, 1, -1) - P(0, -1, 1) + P(0, -1, -1));
              const float dxs = 0.25f * (P(1, 0, 1) - P(1, 0, -1) - P(-1, 0, 1) + P(-1, 0, -1));
              const float dys = 0.25f * (P(1, 1, 0) - P(1, -1, 0) - P(-1, 1, 0) + P(-1, -1, 0));
              const float r0 = -g[0], r1 = -g[1], r2 = -g[2];
              const float m00 = dyy * dss - dys * dys, m01 = dxy * dss - dys * dxs, m02 = dxy * dys - dyy * dxs;
              const float det = dxx * m00 - dxy * m01 + dxs * m02;
              bool ok = std::fabs(det) > 1e-7f;
              const float sd = ok ? det : 1.f;
              const float sn[3] = {(r0 * m00 - dxy * (r1 * dss - dys * r2) + dxs * (r1 * dys - dyy * r2)) / sd,
                                   (dxx * (r1 * dss - dys * r2) - r0 * m01 + dxs * (dxy * r2 - r1 * dxs)) / sd,
                                   (dxx * (dyy * r2 - r1 * dys) - dxy * (dxy * r2 - r1 * dxs) + r0 * m02) / sd};
              if (radius > 0) {
                bool near = false;
                for (int a = std::max(dc - radius, 0); a <= std::min(dc + radius, L - 1); ++a)
                  for (int b = std::max(hc - radius, 0); b <= std::min(hc + radius, H - 1); ++b)
                    for (int e = std::max(wc_ - radius, 0); e <= std::min(wc_ + radius, W - 1); ++e) near = near || is_max(v, a, b, e);
                ok = ok && near;
              }
              valid = ok;
              if (!valid) continue;
              for (int k = 0; k < 3; ++k) s[k] = sn[k];
              gds = g[0] * sn[0] + g[1] * sn[1] + g[2] * sn[2];
              int* pos[3] = {&w, &h, &d};
              const int size[3] = {W, H, L};
              for (int k = 0; k < (allow ? 3 : 2) && valid; ++k) {
                const int nw = *pos[k] + (sn[k] > shift) - (sn[k] < -shift);
                valid = nw >= 1 && nw <= size[k] - 2;
                *pos[k] = std::min(std::max(nw, 0), size[k] - 1);
              }
            }
            valid = valid && std::fabs(s[0]) <= 1.5f && std::fabs(s[1]) <= 1.5f && std::fabs(s[2]) <= 1.5f;
            if (valid) {
              cs = (float)d + s[2];
              cx = (float)w + s[0];
              cy = (float)h + s[1];
            }
            y = src(v, d, h, w) + 0.5f * (valid ? gds : 0.f);
            if (bonus > 0.f) y = y + bonus * (valid ? 1.f : 0.f);
          }
          wc[co] = cs;
          wc[co + L * HW] = cx;
          wc[co + 2 * L * HW] = cy;
          wy[o] = y;
        }
  QuadParams p{};
  p.src = x;
  p.mask = has_mask ? mask.data() : nullptr;
  std::vector<float> cstore, ystore;
  p.coords = aligned(cstore, 3 * n);
  p.y = aligned(ystore, n);
  std::fill(p.coords, p.coords + 3 * n, std::nanf(""));
  std::fill(p.y, p.y + n, std::nanf(""));
  p.sB = sB;
  p.sC = sC;
  p.sL = sL;
  p.ysW = 1;
  p.ysH = W;
  p.ysL = (long long)HW;
  p.ysC = (long long)L * HW;
  p.ysB = (long long)C * L * HW;
  p.C = C;
  p.L = L;
  p.H = H;
  p.W = W;
  p.tiles_x = ceil_div(W, NMS3_TW);
  p.tiles_y = ceil_div(H, NMS3_TH);
  p.tiles = (long long)vols * p.tiles_x * p.tiles_y;
  p.n_iters = n_iters;
  p.radius = radius;
  p.max_shift = shift;
  p.bonus = bonus;
  p.add_bonus = bonus > 0.f;
  p.allow_scale = allow;
  p.refine = refine;
  if (has_mask && radius > 0) emu::launch(grid, dim3(NMS3_NT), [&] { quad_interp3d_kernel<true, true>(p); });
  else if (has_mask) emu::launch(grid, dim3(NMS3_NT), [&] { quad_interp3d_kernel<true, false>(p); });
  else if (radius > 0) emu::launch(grid, dim3(NMS3_NT), [&] { quad_interp3d_kernel<false, true>(p); });
  else emu::launch(grid, dim3(NMS3_NT), [&] { quad_interp3d_kernel<false, false>(p); });
  const std::string what = std::string("quad_interp3d_kernel ") + (radius ? "conv r=" + std::to_string(radius) : std::string("iterative")) +
                           (has_mask ? " mask " : " nms ") + std::to_string(B) + "x" + std::to_string(C) + "x" + std::to_string(L) + "x" +
                           std::to_string(H) + "x" + std::to_string(W) + " n_iters=" + std::to_string(n_iters) + " shift=" + std::to_string(shift) +
                           (allow ? "" : " flat") + (specials ? " special texels" : "") + " grid=" + std::to_string(grid);
  compare_bits_or_nan(what + " (coords)", p.coords, wc.data(), 3 * n);
  compare_bits_or_nan(what + " (y)", p.y, wy.data(), n);
}

// The fixed list (also alone: run_emu --quad): both forms, with and without a mask, radii 1 and 2, n_iters 0, 1 and 5,
// both thresholds and allow_scale_steps, partial edge tiles, D / H / W below 3, special texels, grids that do not divide.
static void test_quad_all() {
  for (int sp = 0; sp < 2; ++sp) {
    test_quad(1, 2, 5, 19, 131, 1, false, 5, 0.6f, 10.f, true, sp, 3);
    test_quad(1, 1, 5, 17, 30, 2, true, 5, 0.3f, 0.f, true, sp, 2);
    test_quad(2, 1, 4, 9, 21, 0, false, 5, 0.3f, 10.f, false, sp, 1);
    test_quad(1, 2, 6, 12, 15, 0, true, 1, 0.6f, 0.f, true, sp, 4);
    test_quad(1, 1, 5, 16, 20, 1, true, 0, 0.3f, 10.f, true, sp, 1);
    test_quad(1, 1, 4, 11, 13, 1, false, 5, 0.3f, 10.f, true, sp, 2);
    test_quad(1, 1, 2, 9, 9, 1, true, 5, 0.6f, 10.f, true, sp, 1);
    test_quad(1, 1, 4, 2, 9, 0, true, 5, 0.6f, 10.f, true, sp, 1);
    test_quad(1, 1, 3, 3, 3, 2, true, 5, 0.3f, 10.f, true, sp, 1);
  }
}

// ------------------------------------------------------------------------------------------ per-patch gradient histograms
// Scalar restatement of SIFTDescriptor.forward / PatchDominantGradientOrientation.forward (kornia/feature/siftdesc.py,
// orientation.py) in the kernels' summation order: the 3 x 3 gradient as every tap FMA'd from 0 in row-major order over a
// replicate border, the reference's fp32 per-pixel ops one rounding each, (b0 == i) * w0 + (b1 == i) * w1 per bin, the
// pooled cells and the histogram bins summed in fp64 in the kernels' order (a cell's window row-major; a bin's pixels lane by
// lane, then the xor butterfly), the block sums per thread then per warp in order.  NaN matches NaN.
static void ph_pixels(const float* patch, int P, const float (*st)[3][3], float eps, const float* weight, int A, bool add_pi,
                      std::vector<int>& b0, std::vector<float>& w0, std::vector<float>& w1) {
  const float pi = 3.14159274101257324219f, two_pi = 6.28318548202514648438f;
  b0.assign(P * P, -1);
  w0.assign(P * P, 0.f);
  w1.assign(P * P, 0.f);
  for (int y = 0; y < P; ++y)
    for (int x = 0; x < P; ++x) {
      float g[2] = {0.f, 0.f};
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
          const float v = patch[std::min(std::max(y + r - 1, 0), P - 1) * P + std::min(std::max(x + c - 1, 0), P - 1)];
          for (int o = 0; o < 2; ++o) g[o] = fmaf(st[o][r][c], v, g[o]);
        }
      const float gx2 = g[0] * g[0], gy2 = g[1] * g[1];
      const float mag = sqrtf((gx2 + gy2) + eps) * weight[y * P + x];
      const float ori = atan2f(g[1], g[0] + eps) + two_pi;
      const float t = (float)A * (add_pi ? ori + pi : ori);
      const float o_big = t / two_pi;
      const float f = floorf(o_big), frac = o_big - f;
      const int e = y * P + x;
      if (!(f != f)) b0[e] = (((int)f % A) + A) % A;
      w0[e] = (1.f - frac) * mag;
      w1[e] = frac * mag;
    }
}
static float ph_value(int b0, float w0, float w1, int i, int A) {
  const int b1 = b0 < 0 ? -1 : (b0 + 1) % A;
  const float a = (b0 == i ? 1.f : 0.f) * w0, b = (b1 == i ? 1.f : 0.f) * w1;
  return a + b;
}
static double butterfly(double* v) {  // the xor butterfly of 32 lanes; every lane ends with lane 0's value
  for (int o = 16; o > 0; o >>= 1) {
    double nv[32];
    for (int l = 0; l < 32; ++l) nv[l] = v[l] + v[l ^ o];
    memcpy(v, nv, sizeof nv);
  }
  return v[0];
}
static double block_sum(const std::vector<double>& part) {  // PH_NT partials
  double s = 0.0;
  for (int w = 0; w < PH_NW; ++w) {
    double lanes[32];
    for (int l = 0; l < 32; ++l) lanes[l] = part[w * 32 + l];
    const double ws = butterfly(lanes);
    s = w == 0 ? ws : s + ws;
  }
  return s;
}
static float divisor(float n) { return n < 1e-12f ? 1e-12f : n; }

static std::vector<float> make_patches(long long N, int P, long long sB, int sH, int specials) {
  std::vector<float> x = randv((size_t)(N * sB));
  if (specials) {
    const float v[5] = {NAN, INFINITY, -INFINITY, -0.f, 1e-40f};
    for (long long n = 1; n < N; n += 3) x[(size_t)(n * sB + (rng() % P) * sH + rng() % P)] = v[rng() % 5];
  }
  return x;
}

static void test_sift(long long N, int P, int A, int S, bool rootsift, float clipval, int specials, unsigned grid) {
  const int K = 2 * (int)(P / (S + 1)), stride = P / S, pad = K / 4, D = A * S * S;
  const int sH = P + 3;
  const long long sB = (long long)sH * P + 5;
  std::vector<float> x = make_patches(N, P, sB, sH, specials), gk = randv(P * P, 0.1f, 1.f), pk = randv(K * K, 0.1f, 1.f);
  std::vector<float> got((size_t)(N * D), -777.f), want((size_t)(N * D));
  SiftParams p{};
  p.src = x.data();
  p.gk = gk.data();
  p.pk = pk.data();
  p.out = got.data();
  p.sB = sB;
  p.sH = sH;
  p.N = N;
  p.P = P;
  p.A = A;
  p.S = S;
  p.K = K;
  p.stride = stride;
  p.pad = pad;
  p.rootsift = rootsift;
  p.clipval = clipval;
  p.eps = 1e-10f;
  emu::launch(grid, dim3(PH_NT), [&] { sift_describe_kernel(p); });
  const GradStencil st = diff_stencil();
  std::vector<float> patch(P * P), desc(D);
  std::vector<int> b0;
  std::vector<float> w0, w1;
  for (long long n = 0; n < N; ++n) {
    for (int y = 0; y < P; ++y)
      for (int xx = 0; xx < P; ++xx) patch[y * P + xx] = x[(size_t)(n * sB + y * sH + xx)];
    ph_pixels(patch.data(), P, st.t, 1e-10f, gk.data(), A, false, b0, w0, w1);
    std::vector<double> part(PH_NT, 0.0);
    for (int c = 0; c < D; ++c) {
      const int i = c / (S * S), cell = c % (S * S), y0 = (cell / S) * stride - pad, x0 = (cell % S) * stride - pad;
      double acc = 0.0;
      for (int ky = 0; ky < K; ++ky)
        for (int kx = 0; kx < K; ++kx) {
          const int y = y0 + ky, xx = x0 + kx;
          const float v = (y >= 0 && y < P && xx >= 0 && xx < P) ? ph_value(b0[y * P + xx], w0[y * P + xx], w1[y * P + xx], i, A) : 0.f;
          acc = fma((double)pk[ky * K + kx], (double)v, acc);
        }
      desc[c] = (float)acc;
      part[c % PH_NT] = fma((double)desc[c], (double)desc[c], part[c % PH_NT]);
    }
    float div = divisor((float)sqrt(block_sum(part)));
    std::fill(part.begin(), part.end(), 0.0);
    for (int c = 0; c < D; ++c) {
      float v = desc[c] / div;
      if (v == v) v = std::min(std::max(v, 0.f), clipval);
      desc[c] = v;
      part[c % PH_NT] = fma((double)v, (double)v, part[c % PH_NT]);
    }
    div = divisor((float)sqrt(block_sum(part)));
    float* out = want.data() + n * D;
    if (rootsift) {
      std::fill(part.begin(), part.end(), 0.0);
      for (int c = 0; c < D; ++c) {
        desc[c] = desc[c] / div;
        part[c % PH_NT] += fabs((double)desc[c]);
      }
      div = divisor((float)block_sum(part));
      for (int c = 0; c < D; ++c) out[c] = sqrtf(desc[c] / div + 1e-10f);
    } else {
      for (int c = 0; c < D; ++c) out[c] = desc[c] / div;
    }
  }
  const std::string what = "sift_describe_kernel N=" + std::to_string(N) + " P=" + std::to_string(P) + " A=" + std::to_string(A) + " S=" +
                           std::to_string(S) + (rootsift ? " rootsift" : " l2") + " clip=" + std::to_string(clipval) +
                           (specials ? " special texels" : "") + " grid=" + std::to_string(grid);
  compare_bits_or_nan(what, got.data(), want.data(), got.size());
}

static void test_orient(long long N, int P, int A, int specials, unsigned grid) {
  const int sH = P + 1;
  const long long sB = (long long)sH * P + 3;
  std::vector<float> x = make_patches(N, P, sB, sH, specials), wt = randv(P * P, 0.1f, 1.f);
  std::vector<float> smooth = {0.1f, 0.2f, 0.4f, 0.2f, 0.1f};
  std::vector<float> got((size_t)N, -777.f), want((size_t)N);
  OriParams p{};
  p.src = x.data();
  p.weighting = wt.data();
  p.smooth = smooth.data();
  p.out = got.data();
  p.sB = sB;
  p.sH = sH;
  p.N = N;
  p.P = P;
  p.A = A;
  p.eps = 1e-8f;
  emu::launch(grid, dim3(PH_NT), [&] { patch_orientation_kernel(p); });
  const GradStencil st = sobel_stencil();
  const float pi = 3.14159274101257324219f, two_pi = 6.28318548202514648438f;
  std::vector<float> patch(P * P), hist(A), sm(A);
  std::vector<int> b0;
  std::vector<float> w0, w1;
  for (long long n = 0; n < N; ++n) {
    for (int y = 0; y < P; ++y)
      for (int xx = 0; xx < P; ++xx) patch[y * P + xx] = x[(size_t)(n * sB + y * sH + xx)];
    ph_pixels(patch.data(), P, st.t, 1e-8f, wt.data(), A, true, b0, w0, w1);
    for (int i = 0; i < A; ++i) {
      double lanes[32];
      for (int l = 0; l < 32; ++l) {
        lanes[l] = 0.0;
        for (int e = l; e < P * P; e += 32) lanes[l] += (double)ph_value(b0[e], w0[e], w1[e], i, A);
      }
      hist[i] = (float)(butterfly(lanes) / (double)(P * P));
    }
    for (int i = 0; i < A; ++i) {
      float acc = 0.f;
      for (int k = 0; k < 5; ++k) acc = fmaf(smooth[k], hist[((i + k - 2) % A + A) % A], acc);
      sm[i] = acc;
    }
    int idx = 0;
    for (int i = 1; i < A && sm[idx] == sm[idx]; ++i)
      if (sm[i] > sm[idx] || sm[i] != sm[i]) idx = i;
    const float c = sm[idx], l = sm[(A + idx - 1) % A], r = sm[(idx + 1) % A];
    const float lr = l - r, half = 0.5f * lr, sum = l + r, c2 = 2.f * c, den = sum - c2, cs = half / den;
    const float t = two_pi * ((float)idx + cs), q = t / (float)A;
    want[n] = -(q - pi);
  }
  const std::string what = "patch_orientation_kernel N=" + std::to_string(N) + " P=" + std::to_string(P) + " A=" + std::to_string(A) +
                           (specials ? " special texels" : "") + " grid=" + std::to_string(grid);
  compare_bits_or_nan(what, got.data(), want.data(), got.size());
}

// Scalar restatement of extract_patches_from_pyramid / extract_patches_simple (kornia/feature/laf.py) in the kernel's op order
// (csrc/laf_patches.cuh): normalisation, scale, level, the level's affine map, then ATen's bilinear 'border' grid_sample
// written out tap by tap.  Levels are random planes of the halving shapes (their values do not matter to the kernel).
static float bilinear_border(const float* s, int h, int w, int sH, float gx, float gy) {
  float ix = (float)(fmaf(gx + 1.f, (float)w, -1.f) * 0.5f), iy = (float)(fmaf(gy + 1.f, (float)h, -1.f) * 0.5f);
  ix = std::fmin((float)(w - 1), std::fmax(ix, 0.f));
  iy = std::fmin((float)(h - 1), std::fmax(iy, 0.f));
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float wx1 = (x0 + 1.f) - ix, wx0 = ix - x0, wy1 = (y0 + 1.f) - iy, wy0 = iy - y0;
  const int xi = (int)x0, yi = (int)y0;
  float acc = 0.f;
  if (xi < w && yi < h) acc = fmaf(s[yi * sH + xi], wx1 * wy1, acc);
  if (xi + 1 < w && yi < h) acc = fmaf(s[yi * sH + xi + 1], wx0 * wy1, acc);
  if (xi < w && yi + 1 < h) acc = fmaf(s[(yi + 1) * sH + xi], wx1 * wy0, acc);
  if (xi + 1 < w && yi + 1 < h) acc = fmaf(s[(yi + 1) * sH + xi + 1], wx0 * wy0, acc);
  return acc;
}

static void test_patches(int B, long long N, int C, int h, int w, int PS, int n_levels, bool normalize, bool select, int row_pad, bool nonfinite,
                         unsigned grid) {
  std::vector<std::vector<float>> store(n_levels);
  LafPatchParams p{};
  int hl = h, wl = w;
  for (int l = 0; l < n_levels; ++l, hl /= 2, wl /= 2) {
    const int sH = wl + (l == 0 ? row_pad : 0);
    const long long sC = (long long)sH * hl + (l == 0 ? 3 : 0), sB = sC * C + (l == 0 ? 7 : 0);
    store[l] = randv((size_t)(sB * B), -1.f, 2.f);
    p.lv[l] = LevelDesc{store[l].data(), sB, sC, hl, wl, sH};
  }
  std::vector<float> laf((size_t)(B * N * 6)), base(PS);
  const int built_top = n_levels;
  for (long long n = 0; n < B * N; ++n) {
    const float u = randv(1, -1.5f, (float)built_top + 1.5f)[0], s = powf(2.f, u) * PS / 2.f, a = randv(1, 0.f, 6.2831853f)[0];
    const float sh = randv(1, -0.3f, 0.3f)[0], r = randv(1, 0.6f, 1.6f)[0];
    float* L = laf.data() + n * 6;
    L[0] = s * cosf(a) * r; L[1] = s * (cosf(a) * sh - sinf(a) / r); L[2] = randv(1, -0.2f, 1.2f)[0] * (w - 1);
    L[3] = s * sinf(a) * r; L[4] = s * (sinf(a) * sh + cosf(a) / r); L[5] = randv(1, -0.2f, 1.2f)[0] * (h - 1);
    if (!normalize)
      for (int k = 0; k < 6; ++k) L[k] /= (float)std::max(1, std::min(h, w) - 1);
    if (nonfinite && n % 4 == 1) L[(n / 4) % 6] = (n % 8 == 1) ? NAN : ((n % 16 == 5) ? -INFINITY : INFINITY);
  }
  for (int j = 0; j < PS; ++j) base[j] = PS > 1 ? (-1.f + 2.f * j / (float)(PS - 1)) * (float)(PS - 1) / (float)PS : 0.f;
  const size_t total = (size_t)(B * N * C * PS * PS);
  std::vector<float> got(total, -777.f), want(total);
  p.laf = laf.data();
  p.base = base.data();
  p.out = got.data();
  p.N = N;
  p.total = B * N;
  p.C = C;
  p.PS = PS;
  p.n_levels = n_levels;
  p.normalize = normalize;
  p.select_level = select;
  if (normalize) {
    p.n_lin = 1.0f / (float)std::min(h - 1, w - 1);
    p.n_tx = (float)(1.0 / (double)(w - 1));
    p.n_ty = (float)(1.0 / (double)(h - 1));
  }
  p.max_clamp = (float)std::max(0, std::min(h, w) / PS - 1);
  emu::launch(grid, dim3(LP_NT), [&] { laf_patches_kernel(p); });
  for (long long n = 0; n < B * N; ++n) {
    const float* L = laf.data() + n * 6;
    float a = L[0], b = L[1], x = L[2], c = L[3], d = L[4], y = L[5];
    if (normalize) {
      a = p.n_lin * a; b = p.n_lin * b; x = p.n_tx * x; c = p.n_lin * c; d = p.n_lin * d; y = p.n_ty * y;
    }
    int lvl = 0;
    if (select) {
      const float m0 = (float)std::min(h - 1, w - 1);
      const float det = ((m0 * a) * (m0 * d) - (m0 * c) * (m0 * b)) + 1e-10f;
      const float sc = (2.0f * sqrtf(fabsf(det))) * (1.0f / (float)PS);
      float l = log2f(sc);
      if (l == l) l = std::fmin(std::fmax(l, 0.f), p.max_clamp);
      const long long L64 = (long long)l;  // the same float -> int64 conversion as the kernel's
      lvl = (L64 >= 0 && L64 < n_levels) ? (int)L64 : -1;
    }
    float* out = want.data() + n * C * PS * PS;
    if (lvl < 0) {
      std::fill(out, out + C * PS * PS, 0.f);
      continue;
    }
    const LevelDesc& lv = p.lv[lvl];
    const float ml = (float)std::min(lv.h - 1, lv.w - 1), wf = (float)(lv.w - 1), hf = (float)(lv.h - 1);
    const float t00 = ml * a, t01 = ml * b, t02 = wf * x, t10 = ml * c, t11 = ml * d, t12 = hf * y, iw = 1.0f / wf, ih = 1.0f / hf;
    for (int i = 0; i < PS; ++i)
      for (int j = 0; j < PS; ++j) {
        const float gx = ((2.0f * (fmaf(base[i], t01, base[j] * t00) + t02)) * iw) - 1.0f;
        const float gy = ((2.0f * (fmaf(base[i], t11, base[j] * t10) + t12)) * ih) - 1.0f;
        for (int ch = 0; ch < C; ++ch)
          out[(size_t)ch * PS * PS + i * PS + j] = bilinear_border(lv.p + (n / N) * lv.sB + ch * lv.sC, lv.h, lv.w, lv.sH, gx, gy);
      }
  }
  const std::string what = "laf_patches_kernel B=" + std::to_string(B) + " N=" + std::to_string(N) + " C=" + std::to_string(C) + " " +
                           std::to_string(h) + "x" + std::to_string(w) + " PS=" + std::to_string(PS) + " levels=" + std::to_string(n_levels) +
                           (normalize ? " norm" : " raw") + (select ? " pyramid" : " simple") + (row_pad ? " strided" : "") +
                           (nonfinite ? " non-finite" : "") + " grid=" + std::to_string(grid);
  compare_bits_or_nan(what, got.data(), want.data(), total);
}

// The fixed list (run_emu --patches): unbuilt levels (fewer levels than the clamp allows), non-finite LAFs, C = 3, PS = 1 and
// 64, odd level sizes, a strided level 0, both functions and normalisations, grids that do not divide the patch count.
static void test_patches_all() {
  test_patches(1, 13, 1, 100, 120, 32, 2, true, true, 0, false, 3);
  test_patches(2, 7, 3, 97, 131, 19, 3, true, true, 0, false, 4);
  test_patches(2, 9, 3, 97, 131, 19, 3, false, true, 5, true, 5);
  test_patches(1, 11, 1, 130, 167, 41, 2, true, true, 0, true, 2);
  test_patches(1, 6, 2, 61, 53, 1, 5, true, true, 9, false, 3);
  test_patches(1, 5, 1, 200, 150, 64, 2, true, true, 0, false, 2);
  test_patches(2, 8, 3, 100, 120, 32, 1, true, false, 4, true, 3);
  test_patches(1, 6, 1, 15, 23, 19, 1, false, true, 0, false, 1);
}

// Scalar restatement of PatchAffineShapeEstimator.forward / LAFAffineShapeEstimator.forward (kornia/feature/affine_shape.py)
// in the kernels' op order (csrc/affine_shape.cuh): the weighted Sobel products summed in fp64 per thread (pixels e = t,
// t + 256, ...) then per warp in order, one rounding of sum / P^2; the degenerate mask and max normalisation; for LAFs
// make_upright, the level and map of test_patches, ATen's bilinear 'border' sampling, ellipse_to_laf's closed-form inverse,
// the rescale and the orientation restore.  NaN matches NaN.
static void aff_moments_ref(const float* patch, int P, const float* wt, float m[3]) {
  const GradStencil st = sobel_stencil();
  std::vector<double> part[3];
  for (int k = 0; k < 3; ++k) part[k].assign(PH_NT, 0.0);
  for (int e = 0; e < P * P; ++e) {
    const int y = e / P, x = e % P;
    float g[2] = {0.f, 0.f};
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        const float v = patch[std::min(std::max(y + r - 1, 0), P - 1) * P + std::min(std::max(x + c - 1, 0), P - 1)];
        for (int o = 0; o < 2; ++o) g[o] = fmaf(st.t[o][r][c], v, g[o]);
      }
    const float gx = g[0] * wt[e], gy = g[1] * wt[e];
    part[0][e % PH_NT] += (double)(gx * gx);
    part[1][e % PH_NT] += (double)(gx * gy);
    part[2][e % PH_NT] += (double)(gy * gy);
  }
  for (int k = 0; k < 3; ++k) m[k] = (float)(block_sum(part[k]) / (double)(P * P));
}
static void aff_tail_ref(float m[3], float eps) {
  const int nb = (m[0] < eps) + (m[1] < eps) + (m[2] < eps);
  const float bad = nb >= 2 ? 1.f : 0.f, keep = 1.f - bad, circ[3] = {1.f, 0.f, 1.f};
  for (int k = 0; k < 3; ++k) m[k] = m[k] * keep + circ[k] * bad;
  float mx = m[0];
  for (int k = 1; k < 3; ++k)
    if (m[k] > mx || m[k] != m[k]) mx = m[k];
  for (int k = 0; k < 3; ++k) m[k] = m[k] / mx;
}
static float scale_ref(float a, float b, float c, float d) { return sqrtf(fabsf((a * d - c * b) + 1e-10f)); }

// Patches: smooth, constant (degenerate), one-direction stripes, anti-correlated ramps (negative b) and special texels.
static void test_patch_affine(long long N, int P, float eps, int specials, unsigned grid) {
  const int sH = P + 2;
  const long long sB = (long long)sH * P + 3;
  std::vector<float> x = make_patches(N, P, sB, sH, specials), wt = randv(P * P, 0.1f, 1.f);
  for (long long n = 0; n < N; ++n)
    for (int y = 0; y < P; ++y)
      for (int xx = 0; xx < P; ++xx) {
        float& v = x[(size_t)(n * sB + y * sH + xx)];
        if (n % 5 == 1) v = 0.25f;                          // constant
        if (n % 5 == 2) v = (float)((xx / 3) % 2);          // vertical stripes: gy = 0
        if (n % 5 == 3) v = 0.1f * (float)(xx - y) + 0.01f * v;  // anti-correlated gradients: b < 0
      }
  std::vector<float> got((size_t)(N * 3), -777.f), want((size_t)(N * 3));
  PatchAffParams p{x.data(), wt.data(), got.data(), sB, sH, N, P, eps};
  emu::launch(grid, dim3(PH_NT), [&] { patch_affine_shape_kernel(p); });
  std::vector<float> patch(P * P);
  for (long long n = 0; n < N; ++n) {
    for (int y = 0; y < P; ++y)
      for (int xx = 0; xx < P; ++xx) patch[y * P + xx] = x[(size_t)(n * sB + y * sH + xx)];
    float m[3];
    aff_moments_ref(patch.data(), P, wt.data(), m);
    aff_tail_ref(m, eps);
    for (int k = 0; k < 3; ++k) want[n * 3 + k] = m[k];
  }
  const std::string what = "patch_affine_shape_kernel N=" + std::to_string(N) + " P=" + std::to_string(P) + " eps=" + std::to_string(eps) +
                           (specials ? " special texels" : "") + " grid=" + std::to_string(grid);
  compare_bits_or_nan(what, got.data(), want.data(), got.size());
}

static void test_laf_affine(int B, long long N, int h, int w, int PS, int n_levels, bool preserve, bool nonfinite, int extra_images,
                            unsigned grid) {
  const int Bimg = B + extra_images;
  std::vector<std::vector<float>> store(n_levels);
  LafAffParams p{};
  int hl = h, wl = w;
  for (int l = 0; l < n_levels; ++l, hl /= 2, wl /= 2) {
    const int sH = wl + (l == 0 ? 3 : 0);
    const long long sB = (long long)sH * hl + (l == 0 ? 5 : 0);
    store[l] = randv((size_t)(sB * Bimg), 0.f, 1.f);
    for (long long i = 0; i < sB * Bimg; i += 7) store[l][i] *= 0.3f;  // texture
    p.lv[l] = LevelDesc{store[l].data(), sB, sB, hl, wl, sH};
  }
  std::vector<float> laf((size_t)(B * N * 6)), base(PS), wt = randv(PS * PS, 0.1f, 1.f);
  for (long long n = 0; n < B * N; ++n) {
    const float u = randv(1, -1.5f, (float)n_levels + 1.5f)[0], s = powf(2.f, u) * PS / 2.f, a = randv(1, 0.f, 6.2831853f)[0];
    const float sh = randv(1, -0.3f, 0.3f)[0], r = randv(1, 0.6f, 1.6f)[0];
    float* L = laf.data() + n * 6;
    L[0] = s * cosf(a) * r; L[1] = s * (cosf(a) * sh - sinf(a) / r); L[2] = randv(1, -0.2f, 1.2f)[0] * (w - 1);
    L[3] = s * sinf(a) * r; L[4] = s * (sinf(a) * sh + cosf(a) / r); L[5] = randv(1, -0.2f, 1.2f)[0] * (h - 1);
    if (nonfinite && n % 4 == 1) L[(n / 4) % 6] = (n % 8 == 1) ? NAN : ((n % 16 == 5) ? -INFINITY : INFINITY);
  }
  for (int j = 0; j < PS; ++j) base[j] = PS > 1 ? (-1.f + 2.f * j / (float)(PS - 1)) * (float)(PS - 1) / (float)PS : 0.f;
  std::vector<float> got((size_t)(B * N * 6), -777.f), want((size_t)(B * N * 6));
  p.laf = laf.data();
  p.base = base.data();
  p.weighting = wt.data();
  p.out = got.data();
  p.N = N;
  p.total = B * N;
  p.PS = PS;
  p.n_levels = n_levels;
  p.n_lin = 1.0f / (float)std::min(h - 1, w - 1);
  p.n_tx = (float)(1.0 / (double)(w - 1));
  p.n_ty = (float)(1.0 / (double)(h - 1));
  p.max_clamp = (float)std::max(0, std::min(h, w) / PS - 1);
  p.eps = 1e-10f;
  p.preserve_orientation = preserve;
  emu::launch(grid, dim3(PH_NT), [&] { laf_affine_shape_kernel(p); });
  std::vector<float> patch(PS * PS);
  for (long long n = 0; n < B * N; ++n) {
    const float* L = laf.data() + n * 6;
    const float a0 = L[0], b0 = L[1], c0 = L[3], d0 = L[4];
    const float det = scale_ref(a0, b0, c0, d0), b2a2 = sqrtf(b0 * b0 + a0 * a0) + 1e-9f;
    float a = det * (b2a2 / det), b = det * 0.f, x = L[2], c = det * ((d0 * b0 + c0 * a0) / (b2a2 * det)), d = det * (det / b2a2), y = L[5];
    a = p.n_lin * a; b = p.n_lin * b; x = p.n_tx * x; c = p.n_lin * c; d = p.n_lin * d; y = p.n_ty * y;
    const float m0 = (float)std::min(h - 1, w - 1);
    const float sc = (2.0f * sqrtf(fabsf(((m0 * a) * (m0 * d) - (m0 * c) * (m0 * b)) + 1e-10f))) * (1.0f / (float)PS);
    float l = log2f(sc);
    if (l == l) l = std::fmin(std::fmax(l, 0.f), p.max_clamp);
    const long long L64 = (long long)l;
    const int lvl = (L64 >= 0 && L64 < n_levels) ? (int)L64 : -1;
    float m[3] = {0.f, 0.f, 0.f};
    if (lvl >= 0) {
      const LevelDesc& lv = p.lv[lvl];
      const float ml = (float)std::min(lv.h - 1, lv.w - 1), wf = (float)(lv.w - 1), hf = (float)(lv.h - 1);
      const float t00 = ml * a, t01 = ml * b, t02 = wf * x, t10 = ml * c, t11 = ml * d, t12 = hf * y, iw = 1.0f / wf, ih = 1.0f / hf;
      for (int i = 0; i < PS; ++i)
        for (int j = 0; j < PS; ++j) {
          const float gx = ((2.0f * (fmaf(base[i], t01, base[j] * t00) + t02)) * iw) - 1.0f;
          const float gy = ((2.0f * (fmaf(base[i], t11, base[j] * t10) + t12)) * ih) - 1.0f;
          patch[i * PS + j] = bilinear_border(lv.p + (n / N) * lv.sB, lv.h, lv.w, lv.sH, gx, gy);
        }
      aff_moments_ref(patch.data(), PS, wt.data(), m);
    }
    aff_tail_ref(m, p.eps);
    const float a11 = sqrtf(fabsf(m[0])), a22 = sqrtf(fabsf(m[2]));
    float den = a11 + a22;
    if (den == den) den = std::fmax(den, 1e-9f);
    const float a21 = m[1] / den, i00 = 1.f / a11, i11 = 1.f / a22, i10 = -(a21 / (a11 * a22)), i01 = 0.f;
    const float coef = det / scale_ref(i00, i01, i10, i11);
    float o[4] = {coef * i00, coef * i01, coef * i10, coef * i11};
    if (preserve) {
      const float pi = 3.14159274101257324219f;
      const float ang = (180.f * atan2f(b0, a0)) / pi - (180.f * atan2f(o[1], o[0])) / pi;
      const float rad = (ang * pi) * (1.f / 180.f), cs = cosf(rad), sn = sinf(rad);
      const float r[2][2] = {{cs, sn}, {-sn, cs}}, lm[2][2] = {{o[0], o[1]}, {o[2], o[3]}};
      for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j) o[2 * i + j] = fmaf(lm[i][1], r[1][j], lm[i][0] * r[0][j]);
    }
    float* out = want.data() + n * 6;
    out[0] = o[0]; out[1] = o[1]; out[2] = L[2]; out[3] = o[2]; out[4] = o[3]; out[5] = L[5];
  }
  const std::string what = "laf_affine_shape_kernel B=" + std::to_string(B) + " N=" + std::to_string(N) + " " + std::to_string(h) + "x" +
                           std::to_string(w) + " PS=" + std::to_string(PS) + " levels=" + std::to_string(n_levels) +
                           (preserve ? " preserve" : " upright") + (nonfinite ? " non-finite" : "") +
                           (extra_images ? " extra images" : "") + " grid=" + std::to_string(grid);
  compare_bits_or_nan(what, got.data(), want.data(), got.size());
}

// The fixed list (run_emu --affine): P = 19, 32, 41, 64 and 3; constant, stripe and negative-b patches, special texels, a
// non-default eps; LAFs at unbuilt levels, non-finite LAFs, both preserve_orientation values, more images than LAF sets,
// grids that do not divide the keypoint count.
static void test_affine_all() {
  test_patch_affine(11, 19, 1e-10f, 0, 3);
  test_patch_affine(7, 32, 1e-10f, 1, 2);
  test_patch_affine(6, 41, 1e-4f, 0, 4);
  test_patch_affine(4, 64, 1e-10f, 1, 3);
  test_patch_affine(5, 3, 1e-10f, 0, 2);
  test_laf_affine(1, 13, 100, 120, 32, 2, true, false, 0, 3);
  test_laf_affine(2, 9, 97, 131, 19, 3, false, true, 0, 4);
  test_laf_affine(1, 11, 130, 167, 41, 2, true, true, 1, 2);
  test_laf_affine(2, 7, 61, 53, 19, 1, true, false, 0, 5);
}

// The fixed lists (run_emu --sift / --orient): every configuration of the reference's tests and the envelope's edges, odd
// batch sizes, grids that do not divide N, batch and row strides that are not P * P and P, special texels.
static void test_sift_all() {
  for (int sp = 0; sp < 2; ++sp) {
    test_sift(7, 41, 8, 4, true, 0.2f, sp, 3);
    test_sift(5, 32, 8, 4, false, 0.1f, sp, 2);
    test_sift(3, 15, 8, 4, true, 0.2f, sp, 1);
    test_sift(9, 19, 5, 3, true, 0.2f, sp, 4);
    test_sift(4, 6, 4, 1, false, 0.2f, sp, 3);
    test_sift(2, 64, 8, 4, true, 0.2f, sp, 1);
    test_sift(3, 32, 16, 8, false, 0.2f, sp, 2);
  }
}
static void test_orient_all() {
  for (int sp = 0; sp < 2; ++sp) {
    test_orient(11, 19, 36, sp, 4);
    test_orient(5, 32, 36, sp, 2);
    test_orient(7, 19, 8, sp, 3);
    test_orient(3, 64, 64, sp, 2);
    test_orient(6, 19, 2, sp, 5);
  }
}

// ------------------------------------------------------------------------------------------ feature responses
// Scalar restatement of kornia/feature/responses.py as this library composes it: spatial_gradient (replicate border,
// row-major FMA over every tap), the products, gaussian_blur2d's row then column pass (reflect border, ascending FMA),
// then one rounding per torch op; torch.min propagates NaN; times sigmas^4.  Compared bit for bit (-0 != +0) with
// corner_vwalk_kernel (Harris, GFTT) and grad_tiled_kernel<GRAD_HESS>.
static const float kSobel1[18] = {-1 / 8.f, 0, 1 / 8.f, -2 / 8.f, 0, 2 / 8.f, -1 / 8.f, 0, 1 / 8.f,
                                  -1 / 8.f, -2 / 8.f, -1 / 8.f, 0, 0, 0, 1 / 8.f, 2 / 8.f, 1 / 8.f};
static const float kDiff1[18] = {0, 0, 0, -0.5f, 0, 0.5f, 0, 0, 0, 0, -0.5f, 0, 0, 0, 0, 0, 0.5f, 0};

template <int KIND>
static void test_corner(int planes, int C, int H, int W, bool diff, int specials, bool sigmas, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  const size_t HW = (size_t)H * W, n = (size_t)planes * HW;
  std::vector<float> xs, os;
  float* x = aligned(xs, n);
  for (size_t i = 0; i < n; ++i) x[i] = randv(1)[0];
  special_texels(x, n, specials);
  const float* st = diff ? kDiff1 : kSobel1;
  float g[CORNER_K], gs = 0.f;
  for (int j = 0; j < CORNER_K; ++j) gs += (g[j] = expf(-0.5f * (float)((j - 3) * (j - 3))));
  for (int j = 0; j < CORNER_K; ++j) g[j] /= gs;
  std::vector<float> s4(planes / C);
  for (auto& v : s4) v = randv(1, 0.5f, 3.f)[0];
  const float k = 0.04f;
  std::vector<float> want(n), prod(3 * HW), row(3 * HW);
  for (int p = 0; p < planes; ++p) {
    const float* xp = x + p * HW;
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        float d[2] = {0.f, 0.f};
        for (int o = 0; o < 2; ++o)
          for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
              d[o] = fmaf(st[(o * 3 + i) * 3 + j], xp[(size_t)fold(y + i - 1, H, KB200_REPLICATE) * W + fold(xx + j - 1, W, KB200_REPLICATE)], d[o]);
        prod[y * W + xx] = d[0] * d[0];
        prod[HW + y * W + xx] = d[1] * d[1];
        prod[2 * HW + y * W + xx] = d[0] * d[1];
      }
    for (int q = 0; q < 3; ++q)
      for (int y = 0; y < H; ++y)
        for (int xx = 0; xx < W; ++xx) {
          float a = 0.f;
          for (int j = 0; j < CORNER_K; ++j) a = fmaf(g[j], prod[q * HW + y * W + fold(xx + j - 3, W, KB200_REFLECT)], a);
          row[q * HW + y * W + xx] = a;
        }
    for (int y = 0; y < H; ++y)
      for (int xx = 0; xx < W; ++xx) {
        float m[3];
        for (int q = 0; q < 3; ++q) {
          float a = 0.f;
          for (int i = 0; i < CORNER_K; ++i) a = fmaf(g[i], row[q * HW + (size_t)fold(y + i - 3, H, KB200_REFLECT) * W + xx], a);
          m[q] = a;
        }
        const float det = m[0] * m[1] - m[2] * m[2], tr = m[0] + m[1], tr2 = tr * tr;
        float r;
        if (KIND == RESP_HARRIS) {
          r = det - k * tr2;
        } else {
          const float sq = sqrtf(fabsf(tr2 - 4.f * det)), e1 = 0.5f * (tr + sq), e2 = 0.5f * (tr - sq);
          r = e1 != e1 ? e1 : e2 != e2 ? e2 : fminf(e1, e2);
        }
        want[p * HW + y * W + xx] = sigmas ? r * s4[p / C] : r;
      }
  }
  CornerParams prm;
  prm.taps = g; prm.kptr = nullptr; prm.s4 = sigmas ? s4.data() : nullptr; prm.out = aligned(os, n);
  prm.planes = planes; prm.C = C; prm.H = H; prm.W = W; prm.k = k;
  for (int e = 0; e < 18; ++e) prm.st[e] = st[e];
  const CUtensorMap map = emu::make_map(x, W, H, planes, VWALK_BW, VWALK_TH + 2, 1), pro = emu::make_map(x, W, H, planes, VWALK_BW, CORNER_K - 1 + 2, 1);
  emu::launch(grid, dim3(256), [&] { corner_vwalk_kernel<KIND>(map, pro, prm); });
  compare_bits_or_nan(std::string("corner_vwalk_kernel ") + (KIND == RESP_HARRIS ? "Harris" : "GFTT") + (diff ? " diff " : " sobel ") + std::to_string(planes) + "x" +
                   std::to_string(H) + "x" + std::to_string(W) + " C=" + std::to_string(C) + (sigmas ? " sigmas" : "") + (specials ? " special texels" : "") +
                   " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager"),
               prm.out, want.data(), n);
}

template <int K>
static void test_hessian(int planes, int C, int H, int W, int specials, bool sigmas, unsigned grid, bool lazy) {
  emu::lazy_tma = lazy;
  const size_t HW = (size_t)H * W, n = (size_t)planes * HW;
  std::vector<float> xs, os;
  float* x = aligned(xs, n);
  for (size_t i = 0; i < n; ++i) x[i] = randv(1)[0];
  special_texels(x, n, specials);
  GradTiledParams p;
  p.H = H; p.W = W; p.planes = planes; p.eps = 0.f; p.C = C;
  auto t = randv(3 * K * K, -1.f, 1.f);
  for (int e = 0; e < 3 * K * K; ++e) p.taps[e] = (e % 4 == 1) ? 0.f : t[e];
  std::vector<float> s4(planes / C);
  for (auto& v : s4) v = randv(1, 0.5f, 3.f)[0];
  p.s4 = sigmas ? s4.data() : nullptr;
  std::vector<float> d(3 * n), want(n);
  ref_filter2d(x, p.taps, 3, d.data(), planes, H, W, K, KB200_REPLICATE);
  for (int pl = 0; pl < planes; ++pl)
    for (size_t i = 0; i < HW; ++i) {
      const float* dp = d.data() + (size_t)pl * 3 * HW;
      const float h = dp[i] * dp[2 * HW + i] - dp[HW + i] * dp[HW + i];
      want[pl * HW + i] = sigmas ? h * s4[pl / C] : h;
    }
  p.out = aligned(os, n);
  const CUtensorMap map = emu::make_map(x, W, H, planes, SEPT_BW, SEPT_TH + K - 1, 1);
  emu::launch(grid, dim3(256), [&] { grad_tiled_kernel<K, 3, GRAD_HESS>(map, p); });
  compare_bits_or_nan("grad_tiled_kernel<GRAD_HESS> K=" + std::to_string(K) + " " + std::to_string(planes) + "x" + std::to_string(H) + "x" + std::to_string(W) +
                   " C=" + std::to_string(C) + (sigmas ? " sigmas" : "") + (specials ? " special texels" : "") + " grid=" + std::to_string(grid) +
                   (lazy ? " lazy" : " eager"),
               p.out, want.data(), n);
}

// The fixed list (also alone: run_emu --responses): edge bands (W = 4, 68, 132), H % 32 in {1, 2} (the last tile's box lies
// entirely below the image), H = W = 4, grids that do not divide the bands (segments that start in the middle of a band),
// both stencil modes, sigmas, and NaN / +-Inf / -0 / subnormal texels.
static void test_responses_all(bool lazy) {
  test_corner<RESP_HARRIS>(3, 3, 70, 132, false, 0, true, 4, lazy);
  test_corner<RESP_HARRIS>(2, 1, 65, 68, true, 1, false, 3, lazy);
  test_corner<RESP_HARRIS>(1, 1, 4, 4, false, 1, true, 1, lazy);
  test_corner<RESP_HARRIS>(2, 2, 97, 200, false, 1, true, 5, lazy);
  test_corner<RESP_GFTT>(3, 3, 66, 132, false, 1, true, 7, lazy);
  test_corner<RESP_GFTT>(2, 1, 33, 4, true, 1, false, 2, lazy);
  test_corner<RESP_GFTT>(1, 1, 34, 68, true, 0, true, 1, lazy);
  test_corner<RESP_GFTT>(4, 2, 129, 72, false, 1, false, 9, lazy);
  test_hessian<5>(3, 3, 70, 132, 1, true, 4, lazy);
  test_hessian<3>(2, 1, 33, 68, 1, false, 3, lazy);
  test_hessian<5>(1, 1, 4, 4, 0, true, 1, lazy);
  test_hessian<3>(2, 2, 65, 260, 1, true, 5, lazy);
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

static void test_undistort(int B, int H, int W, bool lazy, bool strong = false, int specials = 0) {
  emu::lazy_tma = lazy;
  emu::set_smem(remap_smem, sizeof(remap_smem));
  constexpr int C = 3;
  std::vector<float> ss, o1s, o2s, mxs, mys;
  const size_t n = (size_t)B * C * H * W, npix = (size_t)B * H * W;
  float* src = aligned(ss, n);
  for (size_t i = 0; i < n; ++i) src[i] = randv(1)[0];
  special_texels(src, n, specials, (size_t)H * W);
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
    compare_case(specials, "remap_tiled_kernel (verified on hw) vs scalar bilinear " + tag, o1, want.data(), n);
  }
  float* o2 = aligned(o2s, n);
  {
    RemapTiledParams p{src, nullptr, nullptr, o2, B, H, W, H, W, B, 0, lens.data()};
    emu::launch3(grid, dim3(256), [&] { remap_tiled_kernel<3, KB200_ZEROS, true, true>(map, p); });
    compare_case(specials, "remap_tiled_kernel<LENS> (fused undistort) vs maps + remap " + tag, o2, o1, n);
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
static void test_forward(int B, int H, int W, int h, int w, unsigned grid, bool lazy, bool tame, int specials = 0) {
  emu::lazy_tma = lazy;
  emu::set_smem(tma_smem, sizeof(tma_smem));
  constexpr int C = 3;
  const size_t ns = (size_t)B * C * H * W, no = (size_t)B * C * h * w;
  std::vector<float> ss, o1s, o2s;
  float* src = aligned(ss, ns);
  for (size_t i = 0; i < ns; ++i) src[i] = randv(1)[0];
  special_texels(src, ns, specials, (size_t)H * W);
  std::vector<float> m((size_t)B * 9), bx(w), by(h);
  for (int i = 0; i < w; ++i) bx[i] = ((float)i / (float)std::max(w - 1, 1) - 0.5f) * 2.f;
  for (int i = 0; i < h; ++i) by[i] = ((float)i / (float)std::max(h - 1, 1) - 0.5f) * 2.f;
  for (int b = 0; b < B; ++b) {
    const float t = tame ? 0.004f * (b - 1) : (b == 2 ? 0.436f : 0.02f * b);
    const float M[9] = {cosf(t) * (1.f + (tame ? 0.004f : 0.03f) * b), -sinf(t), (tame ? 0.01f : 0.05f) * b - (!tame && b == 1 ? 0.7f : 0.f), sinf(t),
                        cosf(t) * (tame ? 0.995f : 0.97f), tame ? -0.008f : -0.03f, PROJ ? (tame ? 0.004f : 0.02f) : 0.f, PROJ ? (tame ? -0.003f : -0.015f) : 0.f, 1.f};
    memcpy(&m[(size_t)b * 9], M, sizeof(M));
  }
  if (specials >= 2)  // degenerate normalised matrices in place of some samples
    for (int b = 0; b < B; ++b) {
      float* M = &m[(size_t)b * 9];
      switch (rng() % 10) {
        case 0: M[1] = NAN; break;                                          // a NaN entry
        case 1: M[5] = INFINITY; break;                                     // an Inf entry
        case 2: M[2] = 1e8f; break;                                         // pixel coordinates beyond the int range
        case 3: M[2] = -1e30f; break;
        case 4: for (int k = 0; k < 9; ++k) M[k] = 0.f; break;              // zero matrix: 0 / 0 under a projective map
        case 5: M[0] = M[4] = 1e30f; break;                                 // a scale of 1e30
        case 6: M[6] = PROJ ? 1.f : 0.f; M[7] = 0.f; M[8] = PROJ ? 0.f : 1.f; break;  // denominator exactly 0 on the middle column (odd w)
        case 7: for (int k = 0; k < 9; ++k) M[k] *= 1e-20f; break;          // denominator ~1e-20, below the shared-reciprocal window
        case 8: M[0] = -M[0]; M[4] = -M[4]; M[8] = -1.f; break;             // denominator negative everywhere
        default: break;
      }
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
  if (INTERP == KB200_BILINEAR && TW == 64) {
    // the sweep (the run-time work distribution: every run drawn in raster order): same tiles, same results; then the same
    // launch restricted to the footprint class of the wide tile (the producer skips the other class's samples and moves the
    // counter past their runs) against the static deal restricted the same way, with the rotated sample moved to the front
    // twice so that two consecutive samples are skipped
    std::vector<float> o3s, o4s, m2(m);
    float* o3 = aligned(o3s, no);
    float* o4 = aligned(o4s, no);
    if (B >= 3) {
      memcpy(&m2[0], &m[18], 9 * sizeof(float));
      memcpy(&m2[9], &m[18], 9 * sizeof(float));
      memcpy(&m2[18], &m[0], 9 * sizeof(float));
    }
    const std::string tag = " " + std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
    for (size_t i = 0; i < no; ++i) o3[i] = -5.f;
    int counter = 0;
    TmaWarpParams q = p;
    q.out = o3; q.counter = &counter;
    emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2, true>(map, q); });
    compare_case(specials, "warp_fwd_tma<DYN> sweep vs its exact path" + tag, o3, o2, no);
    for (size_t i = 0; i < no; ++i) o3[i] = o4[i] = -5.f;
    counter = 0;
    q.only_class = CLASS_WIDE; q.m = m2.data();
    emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2, true>(map, q); });
    TmaWarpParams r = p;
    r.out = o4; r.only_class = CLASS_WIDE; r.m = m2.data();
    emu::launch(grid, dim3(TMA_THREADS), [&] { warp_fwd_tma<C, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, 2>(map, r); });
    compare_case(specials, "warp_fwd_tma<DYN> sweep wide class only vs the static deal" + tag, o3, o4, no);
  }
  compare_case(specials, std::string("warp_fwd_tma (headline, verified on hw) vs its exact path ") + (PROJ ? "projective " : "affine ") + "interp=" + std::to_string(INTERP) + " pad=" + std::to_string(PAD) + " tile " +
              std::to_string(TW) + "x" + std::to_string(TH) + " " + std::to_string(B) + "x3x" + std::to_string(H) + "x" + std::to_string(W) + " -> " + std::to_string(h) +
              "x" + std::to_string(w) + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager") + (tame ? " tame" : " wild") + (ALIGN ? "" : " align_corners=False"),
          o1, o2, no);
}

// ------------------------------------------------------------------------------------------ tiled warp backward
// Every run is held to the per-element float64 bounds of tests/test_warp_grad_bounds_gpu.py, with the reference computed from
// the kernel's own fp32 coordinates (map_point, unnorm, the border clamp) taken as exact:
//   d/dsrc  |got - ref| <= (4 + n_t) u A_t + tiny     (A_t = sum |w g| over the n_t (pixel, tap) contributions to element t)
//   d/dM    |got - ref| <= u |ref| + (C + 12 + L) u A  (A: the same chain on absolute values; L = 8 max(ceil(w / 64), chunk) + 5)
// Entries whose reference is not finite are compared by class only (specials); entries whose A is not finite have no bound
// and are not compared.
template <bool PROJ, int PAD = KB200_ZEROS, bool ALIGN = true, int C = 3>
static void test_backward(int B, int H, int W, int h, int w, unsigned grid, bool lazy, bool tame = false, int specials = 0) {
  emu::lazy_tma = lazy;
  const size_t ns = (size_t)B * C * H * W, no = (size_t)B * C * h * w;
  std::vector<float> ss, gs, g1s, g2s;
  float* src = aligned(ss, ns);
  float* gout = aligned(gs, no);
  for (size_t i = 0; i < ns; ++i) src[i] = randv(1)[0];
  for (size_t i = 0; i < no; ++i) gout[i] = randv(1, -0.5f, 0.5f)[0];
  // specials 1: special texels in the source, 2: in the upstream gradient.  Without 3e38: the fp64 reference does not overflow
  // where fp32 sums of such terms do, so its classes would differ for a reason that is not the kernel's.
  special_texels(specials == 2 ? gout : src, specials == 2 ? no : ns, specials ? 1 : 0);
  for (float* v : {src, gout})
    for (size_t i = 0, n = v == src ? ns : no; i < n; ++i)
      if (v[i] == 3e38f) v[i] = -2.f;
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
  // scalar reference in double (same fp32 coordinate chain through the kernels' own helpers), its absolute-value chain A and
  // the number of contributions n per source element
  std::vector<double> gsrc_ref(ns, 0.0), gsrc_A(ns, 0.0), gsrc_n((size_t)B * H * W, 0.0), gm_ref((size_t)B * 9, 0.0), gm_A((size_t)B * 9, 0.0);
  const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1);
  const double ux = ALIGN ? Wm1 * 0.5 : W * 0.5, uy = ALIGN ? Hm1 * 0.5 : H * 0.5;
  for (int b = 0; b < B; ++b) {
    Mat3<float> mm;
    mm.load(&m[(size_t)b * 9]);
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        float gx, gy, den;
        map_point<float, PROJ>(mm, bx[x], by[y], gx, gy, den);
        float ix = unnorm<ALIGN>(gx, Wm1, (float)W), iy = unnorm<ALIGN>(gy, Hm1, (float)H);
        if (!(fabsf(ix) < 1.0e9f && fabsf(iy) < 1.0e9f)) continue;
        double px = 1, py = 1;
        if (PAD == KB200_BORDER) {
          if (ix <= 0.f) { ix = 0.f; px = 0; } else if (ix >= Wm1) { ix = Wm1; px = 0; }
          if (iy <= 0.f) { iy = 0.f; py = 0; } else if (iy >= Hm1) { iy = Hm1; py = 0; }
        }
        const double x0f = floor((double)ix), y0f = floor((double)iy);
        const double wx0 = (double)ix - x0f, wx1 = 1.0 - wx0, wy0 = (double)iy - y0f, wy1 = 1.0 - wy0;
        const int x0 = (int)x0f, y0 = (int)y0f;
        auto ok = [&](int yy, int xx) { return yy >= 0 && yy < H && xx >= 0 && xx < W; };
        double gix = 0, giy = 0, aix = 0, aiy = 0;
        for (int c = 0; c < C; ++c) {
          const double go = gout[(((size_t)b * C + c) * h + y) * w + x];
          const float* sp = src + ((size_t)b * C + c) * H * W;
          double* gp = gsrc_ref.data() + ((size_t)b * C + c) * H * W;
          double* ap = gsrc_A.data() + ((size_t)b * C + c) * H * W;
          double* np = gsrc_n.data() + (size_t)b * H * W;
          auto v = [&](int yy, int xx) { return ok(yy, xx) ? (double)sp[(size_t)yy * W + xx] : 0.0; };
          auto tap = [&](int yy, int xx, double wt) {
            if (!ok(yy, xx)) return;
            gp[(size_t)yy * W + xx] += wt * go;
            ap[(size_t)yy * W + xx] += wt * fabs(go);
            if (c == 0) np[(size_t)yy * W + xx] += 1;
          };
          tap(y0, x0, wx1 * wy1); tap(y0, x0 + 1, wx0 * wy1); tap(y0 + 1, x0, wx1 * wy0); tap(y0 + 1, x0 + 1, wx0 * wy0);
          gix += go * ((v(y0, x0 + 1) - v(y0, x0)) * wy1 + (v(y0 + 1, x0 + 1) - v(y0 + 1, x0)) * wy0);
          giy += go * ((v(y0 + 1, x0) - v(y0, x0)) * wx1 + (v(y0 + 1, x0 + 1) - v(y0, x0 + 1)) * wx0);
          aix += fabs(go) * ((fabs(v(y0, x0 + 1)) + fabs(v(y0, x0))) * wy1 + (fabs(v(y0 + 1, x0 + 1)) + fabs(v(y0 + 1, x0))) * wy0);
          aiy += fabs(go) * ((fabs(v(y0 + 1, x0)) + fabs(v(y0, x0))) * wx1 + (fabs(v(y0 + 1, x0 + 1)) + fabs(v(y0, x0 + 1))) * wx0);
        }
        const double rden = PROJ ? 1.0 / (double)den : 1.0;
        const double ax = gix * ux * px * rden, ay = giy * uy * py * rden, az = -(ax * gx + ay * gy);
        const double bax = aix * ux * px * fabs(rden), bay = aiy * uy * py * fabs(rden), baz = bax * fabs(gx) + bay * fabs(gy);
        double* g = &gm_ref[(size_t)b * 9];
        double* a = &gm_A[(size_t)b * 9];
        g[0] += ax * bx[x]; g[1] += ax * by[y]; g[2] += ax;
        g[3] += ay * bx[x]; g[4] += ay * by[y]; g[5] += ay;
        a[0] += bax * fabs(bx[x]); a[1] += bax * fabs(by[y]); a[2] += bax;
        a[3] += bay * fabs(bx[x]); a[4] += bay * fabs(by[y]); a[5] += bay;
        if (PROJ) {
          g[6] += az * bx[x]; g[7] += az * by[y]; g[8] += az;
          a[6] += baz * fabs(bx[x]); a[7] += baz * fabs(by[y]); a[8] += baz;
        }
      }
  }
  const int nstrips = B * ceil_div(h, 32), max_segs = nstrips / (int)grid + 2;
  const size_t rows = (size_t)grid * max_segs;
  constexpr int CHUNK = 3;  // tiles per chunk of the run-time deal here
  long long exact[6] = {0, 0, 0, 0, 0, 0};
  // version 2: column-pair lanes, 3: stride-1 lanes, 5: stride-1 lanes drawn at run time; need: 3 both, 1 d/dsrc only, 2 d/dM only
  auto run = [&](int version, int need, float* gsrc, std::vector<double>& gm) {
    emu_exact_path_pixels = 0;
    for (size_t i = 0; i < ns; ++i) gsrc[i] = 0.f;
    std::vector<float> records(rows * 8 * 9, 0.f);
    std::vector<int> rb(rows, -7);
    TmaBwdParams p{};
    p.gout = gout; p.src = src; p.m = m.data(); p.bx = bx.data(); p.by = by.data(); p.gsrc = (need & 1) ? gsrc : nullptr;
    p.records = records.data(); p.record_batch = rb.data();
    p.B = B; p.H = H; p.W = W; p.h = h; p.w = w; p.Bm = B; p.max_segs = max_segs;
    const CUtensorMap mgsrc = emu::make_map(gsrc, W, H, B * C, 72, BWD_SH, C), mgout = emu::make_map(gout, w, h, B * C, 64, 32, C);
    emu::set_smem(bwd2_smem, sizeof(bwd2_smem));
    const CUtensorMap mwin = emu::make_map(src, W, H, B * C, 72, BWD_SH, C);
    int counter = 0;
    size_t use_rows = rows;
    if (version == 5) {  // the run-time work distribution: one record row per chunk
      p.counter = &counter;
      p.chunk_tiles = CHUNK;
      use_rows = (size_t)B * ceil_div(h, 32) * ceil_div(ceil_div(w, 64), CHUNK);
      records.assign(use_rows * 8 * 9, 0.f);
      rb.assign(use_rows, -7);
      p.records = records.data(); p.record_batch = rb.data();
      emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, PAD, PROJ, ALIGN, true, true, true, true>(mwin, mgsrc, mgout, p); });
    } else if (version == 2) {
      emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, PAD, PROJ, ALIGN, true, true, false>(mwin, mgsrc, mgout, p); });
    } else if (need == 1) {
      emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, PAD, PROJ, ALIGN, true, false, true>(mwin, mgsrc, mgout, p); });
    } else if (need == 2) {
      emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, PAD, PROJ, ALIGN, false, true, true>(mwin, mgsrc, mgout, p); });
    } else {
      emu::launch(grid, dim3(BWD_THREADS), [&] { warp_bwd_tma2<C, PAD, PROJ, ALIGN, true, true, true>(mwin, mgsrc, mgout, p); });
    }
    exact[version] = emu_exact_path_pixels;
    gm.assign((size_t)B * 9, 0.0);
    if (need & 2)
      for (size_t r = 0; r < use_rows; ++r)
        if (rb[r] >= 0)
          for (int wv = 0; wv < 8; ++wv)
            for (int k = 0; k < 9; ++k) gm[(size_t)rb[r] * 9 + k] += (double)records[(r * 8 + wv) * 9 + k];
  };
  const std::string tag = std::string(PROJ ? "projective " : "affine     ") + std::to_string(B) + "x" + std::to_string(C) + "x" + std::to_string(H) + "x" +
                          std::to_string(W) + " -> " + std::to_string(h) + "x" + std::to_string(w) + (PAD == KB200_BORDER ? " border" : " zeros") +
                          (ALIGN ? "" : " align_corners=False") + " grid=" + std::to_string(grid) + (lazy ? " lazy" : " eager");
  const double u = 1.0 / 16777216.0, tiny = 1.17549435e-38;
  const double Lrun = 8.0 * std::max(ceil_div(w, 64), CHUNK) + 5, cpix = C + 12;
  auto check = [&](const char* name, const float* g, const std::vector<double>& gm, int need) {
    auto cls = [](double v) { return v != v ? 3 : v == INFINITY ? 1 : v == -INFINITY ? 2 : 0; };
    size_t bad = 0, out_src = 0, out_m = 0;
    double r_src = 0, r_m = 0;  // largest |got - ref| / (u A)
    if (need & 1)
      for (size_t i = 0; i < ns; ++i) {
        if (cls(g[i]) != cls(gsrc_ref[i])) { ++bad; continue; }
        if (cls(g[i])) continue;
        const double A = gsrc_A[i], n = gsrc_n[(i / ((size_t)C * H * W)) * H * W + i % ((size_t)H * W)];
        const double err = fabs((double)g[i] - gsrc_ref[i]);
        if (std::isfinite(A)) {
          if (err > (4 + n) * u * A + tiny) ++out_src;
          if (A > 0) r_src = std::max(r_src, err / (u * A));
        }
      }
    if (need & 2)
      for (size_t i = 0; i < gm.size(); ++i) {
        if (cls(gm[i]) != cls(gm_ref[i])) { ++bad; continue; }
        if (cls(gm[i])) continue;
        const double err = fabs(gm[i] - gm_ref[i]), A = gm_A[i];
        if (std::isfinite(A)) {
          if (err > u * fabs(gm_ref[i]) + (cpix + Lrun) * u * A + tiny) ++out_m;
          if (A > 0) r_m = std::max(r_m, err / (u * A));
        }
      }
    const bool ok = bad == 0 && out_src == 0 && out_m == 0;
    printf("%s %-58s %s%s  specials=%d: %zu class mismatches, d/dsrc %zu out of bound (max %.3g u A), d/dM %zu out of bound (max %.3g u A)\n",
           ok ? "ok  " : "FAIL", name, tag.c_str(), need == 1 ? " d/dsrc only" : need == 2 ? " d/dM only" : "", specials, bad, out_src, r_src, out_m, r_m);
    if (!ok) ++failures;
  };
  float* g1 = aligned(g1s, ns);
  float* g2 = aligned(g2s, ns);
  std::vector<double> gm1, gm2;
  run(2, 3, g1, gm1);
  run(3, 3, g2, gm2);
  printf("     pixels on the exact (global-memory) path: warp_bwd_tma2 %lld, stride-1 lanes %lld of %d\n", exact[2], exact[3], B * h * w);
  check("warp_bwd_tma2 (per-warp pipelines) vs fp64 scalar backward", g1, gm1, 3);
  check("warp_bwd_tma2<STRIDE1> (conflict-free lanes) vs fp64 scalar backward", g2, gm2, 3);
  run(3, 1, g2, gm2);
  check("warp_bwd_tma2<STRIDE1> (conflict-free lanes) vs fp64 scalar backward", g2, gm2, 1);
  run(3, 2, g2, gm2);
  check("warp_bwd_tma2<STRIDE1> (conflict-free lanes) vs fp64 scalar backward", g2, gm2, 2);
  if (C == 3) {  // the dispatcher takes the run-time deal for RGB only
    run(5, 3, g2, gm2);
    check("warp_bwd_tma2<STRIDE1, DYN> (work drawn at run time) vs fp64 scalar backward", g2, gm2, 3);
  }
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

// The special-value list (also alone: run_emu --specials): NaN / +-Inf / -0 / subnormal / 1e-38 / 3e38 texels and a plane of
// -0 through every tiled kernel, compared bit for bit (-0 != +0); the headline forward kernel (both tile shapes, every
// interpolation) also under degenerate matrices; the tiled backward with special texels and special upstream gradients.
static void test_specials_all(bool lazy) {
  for (int sp = 1; sp <= 2; ++sp) {
    test_sepfilter<11, KB200_REFLECT>(2, 3, 70, 132, 5, lazy, sp);
    test_sepfilter<3, KB200_CONSTANT>(1, 2, 33, 68, 2, lazy, sp);
    test_sepfilter<17, KB200_REPLICATE>(1, 2, 97, 140, 3, lazy, sp);
    test_filter2d<3, KB200_REFLECT>(3, 70, 132, 4, lazy, sp);
    test_filter2d<5, KB200_CONSTANT>(2, 33, 68, 2, lazy, sp);
    test_filter2d<7, KB200_REPLICATE>(2, 40, 72, 3, lazy, sp);
    test_pyrdown<KB200_REFLECT>(3, 70, 132, 4, lazy, sp);
    test_pyrdown<KB200_CONSTANT>(2, 34, 68, 3, lazy, sp);
    test_gradient<3, 2, false>(3, 70, 132, 4, lazy, sp);
    test_gradient<3, 2, true>(2, 33, 260, 3, lazy, sp);
    test_gradient<5, 3, false>(2, 97, 136, 5, lazy, sp);
    test_ssim<11>(3, 70, 132, 4, lazy, sp);
    test_ssim<7>(2, 33, 68, 3, lazy, sp);
    test_undistort(2, 70, 132, lazy, false, sp);
    test_undistort(2, 97, 200, lazy, true, sp);
    test_forward<true, KB200_ZEROS, 64, 32, 72, 40>(3, 70, 132, 50, 101, 2, lazy, false, sp);
    test_forward<true, KB200_ZEROS, 64, 32, 72, 40>(4, 96, 200, 96, 199, 3, lazy, true, sp);
    test_forward<false, KB200_BORDER, 64, 32, 72, 40>(3, 64, 128, 70, 133, 4, lazy, true, sp);
    test_forward<true, KB200_REFLECTION, 64, 32, 72, 40>(3, 70, 132, 70, 131, 3, lazy, false, sp);
    test_forward<true, KB200_FILL, 64, 32, 72, 40>(3, 70, 132, 64, 121, 2, lazy, true, sp);
    test_forward<true, KB200_ZEROS, 32, 32, 56, 56>(3, 70, 132, 70, 131, 3, lazy, false, sp);
    test_forward<true, KB200_REFLECTION, 32, 32, 56, 56>(3, 70, 132, 70, 131, 2, lazy, true, sp);
    test_forward<true, KB200_ZEROS, 64, 32, 72, 40, KB200_NEAREST>(3, 70, 132, 70, 131, 3, lazy, true, sp);
    test_forward<true, KB200_BORDER, 64, 32, 72, 40, KB200_BICUBIC>(3, 70, 132, 70, 131, 2, lazy, true, sp);
    test_forward<false, KB200_REFLECTION, 64, 32, 72, 40, KB200_BICUBIC>(3, 64, 128, 70, 133, 3, lazy, false, sp);
    test_backward<true>(3, 70, 132, 70, 132, 2, lazy, false, sp);
    test_backward<false>(3, 64, 128, 50, 96, 3, lazy, true, sp);
  }
}

static void fuzz(int rounds) {
  std::mt19937 g(20260923);
  auto pick = [&](int lo, int hi) { return lo + (int)(g() % (unsigned)(hi - lo + 1)); };
  std::mt19937 go(20261017);  // the octave cases draw from their own stream, so the other cases stay what they were
  auto opick = [&](int lo, int hi) { return lo + (int)(go() % (unsigned)(hi - lo + 1)); };
  std::mt19937 gn(20261018);  // and the non-maximum-suppression cases from theirs
  auto npick = [&](int lo, int hi) { return lo + (int)(gn() % (unsigned)(hi - lo + 1)); };
  std::mt19937 gq(20261019);  // and the sub-pixel refinement cases from theirs
  auto qpick = [&](int lo, int hi) { return lo + (int)(gq() % (unsigned)(hi - lo + 1)); };
  std::mt19937 gs(20261020);  // and the gradient-histogram cases from theirs
  for (int r = 0; r < rounds; ++r) {
    if (r % 10 == 9) {  // ScalePyramid octave: any chain, both stage-0 modes, sides from the largest tap count up, any grid
      const int which = opick(0, 4), planes = opick(1, 2), sp = opick(0, 2);
      const unsigned grid = (unsigned)opick(1, 12);
      const int kmax = which == 1 || which == 4 ? 21 : 25;
      const int H = opick(kmax, 120), W = 4 * opick((kmax + 3) / 4, 70);
      if (which == 0) test_octave<OctDefault>(planes, H, W, sp, grid);
      else if (which == 1) test_octave<OctDetector>(planes, H, W, sp, grid);
      else if (which == 2) test_octave<OctDouble>(planes, H, W, sp, grid);
      else if (which == 3) test_octave<OctCopy6>(planes, H, W, sp, grid);
      else test_octave<OctCopy5>(planes, H, W, sp, grid);
    }
    if (r % 10 == 4) {  // non-maximum suppression: any K and form, any shape (odd widths, sides below K), 3-D modes, any grid
      const int H = npick(1, 80), W = npick(1, 140), sp = npick(0, 1);
      const unsigned grid = (unsigned)npick(1, 9);
      switch (npick(0, 9)) {
        case 0: test_nms2d_both<3>(npick(1, 2), npick(1, 2), H, W, sp, grid); break;
        case 1: test_nms2d_both<5>(1, npick(1, 2), H, W, sp, grid); break;
        case 2: test_nms2d_both<7>(1, 1, H, W, sp, grid); break;
        case 3: test_nms2d_both<9>(1, npick(1, 2), H, W, sp, grid); break;
        case 4: test_nms2d_both<15>(npick(1, 2), 1, H, W, sp, grid); break;
        case 5: test_nms2d_both<21>(1, 1, H, W, sp, grid); break;
        case 6: test_nms2d_both<31>(1, 1, H, W, sp, grid); break;
        case 7: test_nms3d<NMS3_MAX_MASK>(npick(1, 2), npick(1, 2), npick(1, 5), H / 2 + 1, W, sp, grid); break;
        case 8: test_nms3d<NMS3_MAX_VALUES>(1, npick(1, 2), npick(1, 5), H / 2 + 1, W, sp, grid); break;
        default: test_nms3d<NMS3_MINMAX>(npick(1, 2), npick(1, 2), npick(1, 6), H / 2 + 1, W, sp, grid); break;
      }
    }
    if (r % 10 == 7) {  // sub-pixel refinement: either form, with or without a mask, any parameters, shape and grid
      const int n_iters = qpick(0, 6), radius = qpick(0, 2), mask = qpick(0, 1), allow = qpick(0, 1), sp = qpick(0, 1);
      const float shift = qpick(0, 1) ? 0.6f : 0.3f, bonus = qpick(0, 1) ? 10.f : 0.f;
      test_quad(qpick(1, 2), qpick(1, 2), qpick(1, 6), qpick(1, 24), qpick(1, 140), radius, mask, n_iters, shift, bonus, allow, sp,
                (unsigned)qpick(1, 9));
    }
    if (r % 10 == 2) {  // per-patch gradient histograms: any envelope configuration, batch size and grid
      auto spick = [&](int lo, int hi) { return lo + (int)(gs() % (unsigned)(hi - lo + 1)); };
      static const int cfg[7][3] = {{41, 8, 4}, {32, 8, 4}, {15, 8, 4}, {19, 5, 3}, {6, 4, 1}, {64, 8, 4}, {32, 16, 8}};
      const int* c = cfg[spick(0, 6)];
      test_sift(spick(1, 9), c[0], c[1], c[2], c[0] != 6 && spick(0, 1), spick(0, 1) ? 0.2f : 0.1f, spick(0, 1), (unsigned)spick(1, 7));
      test_orient(spick(1, 9), spick(0, 1) ? 19 : 32, spick(0, 1) ? 36 : spick(2, 64), spick(0, 1), (unsigned)spick(1, 7));
    }
    const int H = pick(1, 110), W = 4 * pick(1, 70), planes = pick(1, 4), lazy = pick(0, 1);
    const unsigned grid = (unsigned)pick(1, 9);
    switch (pick(0, 50)) {
      case 47:
      case 48: {  // special texels (and degenerate matrices) through the tiled filters and the headline forward kernel
        const int sp = pick(1, 2);
        const int which = pick(0, 5);
        if (which == 0 && H > 5 && W > 5) test_sepfilter<11, KB200_REFLECT>(1, planes, H, W, grid, lazy, sp);
        else if (which == 1) test_filter2d<5, KB200_CONSTANT>(planes, H, W, grid, lazy, sp);
        else if (which == 2 && H > 2) test_gradient<5, 3, false>(planes, H, W, grid, lazy, sp);
        else if (which == 3 && H > 1) test_forward<true, KB200_ZEROS, 64, 32, 72, 40>(3, H, W, std::max(1, H - pick(0, 5)), std::max(4, W - pick(0, 3)), grid, lazy, pick(0, 1), sp);
        else if (which == 4 && H > 1) test_forward<true, KB200_REFLECTION, 32, 32, 56, 56, KB200_BICUBIC>(3, H, W, H, std::max(4, W - 1), grid, lazy, pick(0, 1), sp);
        else if (H > 3 && W > 3) test_ssim<7>(planes, H, W, grid, lazy, sp);
        break;
      }
      case 49:
      case 50: {  // remap / fused undistort and the tiled backward with special values
        const int sp = pick(1, 2);
        if (pick(0, 1) && H > 1) test_undistort(pick(1, 2), H, W, lazy, pick(0, 1), sp);
        else if (H > 1 && W > 4) test_backward<true>(3, H, W, std::max(2, H - pick(0, 3)), std::max(8, W - 4 * pick(0, 2)), grid, lazy, pick(0, 1), sp);
        break;
      }
      case 44:
      case 45:
      case 46: {  // feature responses: Harris / GFTT / Hessian, both stencil modes, C 1..3, sigmas, special texels
        const int C = pick(1, 3), B = pick(1, 2), specials = pick(0, 1), sig = pick(0, 1), diff = pick(0, 1);
        const int Hh = std::max(H, 4), Wh = std::max(W, 4);
        const int which = pick(0, 3);
        if (which == 0) test_corner<RESP_HARRIS>(B * C, C, Hh, Wh, diff, specials, sig, grid, lazy);
        else if (which == 1) test_corner<RESP_GFTT>(B * C, C, Hh, Wh, diff, specials, sig, grid, lazy);
        else if (which == 2) test_hessian<3>(B * C, C, Hh, Wh, specials, sig, grid, lazy);
        else test_hessian<5>(B * C, C, Hh, Wh, specials, sig, grid, lazy);
        break;
      }
      case 41:
      case 42:
      case 43: {  // zero-skipping filter2d: any odd K 9..31, kernel kind, special texels, Bk 1 / B / cycling
        const int K = 2 * pick(4, 15) + 1, B = pick(1, 4), C = pick(1, 2), kind = pick(0, 5), specials = pick(0, 3);
        const int Bk = pick(0, 2) == 0 ? 1 : pick(0, 1) ? B : pick(1, 3);
        const int h = (K - 1) / 2;
        const int Hh = std::max(H, h + 1), Wh = std::max(W, 4 * ((h + 4) / 4));
        if (g() % 3 == 0) test_taps<KB200_CONSTANT>(K, B, C, H, W, Bk, kind, specials, grid, lazy);
        else if (g() % 2) test_taps<KB200_REFLECT>(K, B, C, Hh, Wh, Bk, kind, specials, grid, lazy);
        else test_taps<KB200_REPLICATE>(K, B, C, Hh, Wh, Bk, kind, specials, grid, lazy);
        break;
      }
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
  if (argc == 2 && std::string(argv[1]) == "--taps") {
    for (int lazy = 0; lazy < 2; ++lazy) test_taps_all(lazy);
    printf("%s: %d failing comparisons (filter2d_taps_kernel, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--responses") {
    for (int lazy = 0; lazy < 2; ++lazy) test_responses_all(lazy);
    printf("%s: %d failing comparisons (feature responses, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--octave") {
    test_octave_all();
    printf("%s: %d failing comparisons (ScalePyramid octave, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--nms") {
    test_nms_all();
    printf("%s: %d failing comparisons (non-maximum suppression, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--quad") {
    test_quad_all();
    printf("%s: %d failing comparisons (sub-pixel refinement, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc >= 2 && (std::string(argv[1]) == "--sift" || std::string(argv[1]) == "--orient")) {
    for (int a = 1; a < argc; ++a) {
      if (std::string(argv[a]) == "--sift") test_sift_all();
      if (std::string(argv[a]) == "--orient") test_orient_all();
    }
    printf("%s: %d failing comparisons (per-patch gradient histograms, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures,
           emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--patches") {
    test_patches_all();
    printf("%s: %d failing comparisons (LAF patch extraction, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--affine") {
    test_affine_all();
    printf("%s: %d failing comparisons (affine shape, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
  }
  if (argc == 2 && std::string(argv[1]) == "--specials") {
    for (int lazy = 0; lazy < 2; ++lazy) test_specials_all(lazy);
    printf("%s: %d failing comparisons (special values, %d of them bit-level)\n", failures ? "FAILED" : "PASSED", failures, emu_strict_failures);
    return failures ? 1 : 0;
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
    test_taps_all(lazy);
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
    test_backward<true, KB200_BORDER>(3, 70, 132, 70, 132, 2, lazy);
    test_backward<false, KB200_BORDER, false>(3, 64, 128, 50, 96, 3, lazy);
    test_backward<true, KB200_ZEROS, false>(3, 40, 72, 66, 132, 4, lazy);
    test_backward<true, KB200_ZEROS, true, 1>(3, 70, 132, 70, 132, 2, lazy);
    test_backward<false, KB200_BORDER, false, 1>(3, 96, 200, 96, 200, 3, lazy, true);
  }
  printf("%s: %d failing comparisons, %lld TMA loads, %lld TMA reduce-adds, %lld CTA barriers and %lld warp rendezvous emulated\n",
         failures ? "FAILED" : "PASSED", failures, emu::n_tma, emu::n_reduce, emu::n_barriers, emu::n_wsync);
  return failures ? 1 : 0;
}
