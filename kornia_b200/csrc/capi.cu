// kornia_b200 -- extern "C" entry points (include/kornia_b200.h) and kernel dispatch.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "filter_generic.cuh"
#include "prelude.cuh"
#include "warp_generic.cuh"
#include "warp_tma.cuh"
#include "warp_bwd_tma.cuh"
#include "sepfilter_tiled.cuh"
#include "filter2d_tiled.cuh"
#include "filter2d_taps.cuh"
#include "remap_tiled.cuh"
#include "gradient.cuh"
#include "ssim_vwalk.cuh"
#include "corner_vwalk.cuh"
#include "octave_vwalk.cuh"
#include "nms.cuh"
#include "quad_interp.cuh"
#include "gradient_tiled.cuh"

namespace kb200 {

static thread_local char g_err[512] = "";
static thread_local const char* g_variant = "none";
static thread_local int g_warp_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---------------------------------------------------------------- kernel-selection switches (common.cuh: enum Option)
// One row per switch, keyed by its enum value: the loader and the name lookup never depend on the order of the rows.
static const struct {
  Option opt;
  const char* name;
  int value;  // default, unless KB200_<NAME> is set
} OPTIONS[] = {
    {OPT_TMA, "tma", 1},
    {OPT_TILED_FILTER, "tiled_filter", 1},
    {OPT_SQUARE_TILES, "square_tiles", 1},
    {OPT_TILED_GRADIENT, "tiled_gradient", 1},
    {OPT_U8_TILED, "u8_tiled", 1},
    {OPT_BWD_STRIDE1, "bwd_stride1", 1},
    {OPT_DYN_SCHED, "dyn_sched", 1},
};
static_assert(sizeof(OPTIONS) / sizeof(OPTIONS[0]) == OPT_COUNT, "one OPTIONS row per Option");
static int g_options[OPT_COUNT];
static const bool g_options_ready = [] {  // once, when the library is loaded: KB200_<NAME>=<int> overrides the default
  for (const auto& row : OPTIONS) {
    char env[64] = "KB200_";
    size_t n = strlen(env);
    for (const char* c = row.name; *c && n + 1 < sizeof(env); ++c) env[n++] = (char)((*c >= 'a' && *c <= 'z') ? *c - 32 : *c);
    env[n] = 0;
    const char* v = getenv(env);
    g_options[row.opt] = (v && v[0]) ? atoi(v) : row.value;
  }
  return true;
}();
int option(Option o) { return __atomic_load_n(&g_options[o], __ATOMIC_RELAXED); }
static int option_index(const char* name) {
  for (const auto& row : OPTIONS)
    if (name && strcmp(name, row.name) == 0) return row.opt;
  return -1;
}

static int post_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

// blockIdx.z carries the sample / plane index; CUDA caps gridDim.z at 65535
constexpr int MAX_Z = 65535;

// ------------------------------------------------------------------------------------------
// warp / remap dispatch
// ------------------------------------------------------------------------------------------
template <typename T, int INTERP, int PAD, int KIND>
static int launch_warp_fwd(WarpParams<T> p, cudaStream_t st) {
  const dim3 block(GEN_BX, GEN_BY);
  const int B = p.B;
  for (int b0 = 0; b0 < B; b0 += MAX_Z) {
    WarpParams<T> q = p;
    q.B = min(MAX_Z, B - b0);
    q.src = p.src + (size_t)b0 * p.C * p.H * p.W;
    q.out = p.out + (size_t)b0 * p.C * p.h * p.w;
    if (KIND == KIND_REMAP) {
      if (p.Bm != 1) {
        q.map_x = p.map_x + (size_t)b0 * p.h * p.w;
        q.map_y = p.map_y + (size_t)b0 * p.h * p.w;
      }
    } else if (p.Bm != 1) {
      q.m = p.m + (size_t)b0 * 9;
    }
    const dim3 grid(ceil_div(p.w, GEN_BX), ceil_div(p.h, GEN_BY), q.B);
    warp_fwd_generic<T, INTERP, PAD, KIND><<<grid, block, 0, st>>>(q);
  }
  return post_launch("warp_forward");
}

template <typename T, int INTERP, int PAD, int KIND>
static int launch_warp_bwd(WarpGradParams<T> g, cudaStream_t st) {
  const dim3 block(GEN_BX, GEN_BY);
  const WarpParams<T>& p = g.p;
  const int B = p.B;
  const size_t nblk = (size_t)ceil_div(p.w, GEN_BX) * ceil_div(p.h, GEN_BY);
  for (int b0 = 0; b0 < B; b0 += MAX_Z) {
    WarpGradParams<T> q = g;
    q.p.B = min(MAX_Z, B - b0);
    q.p.src = p.src + (size_t)b0 * p.C * p.H * p.W;
    q.gout = g.gout + (size_t)b0 * p.C * p.h * p.w;
    if (g.gsrc) q.gsrc = g.gsrc + (size_t)b0 * p.C * p.H * p.W;
    if (g.partial) q.partial = g.partial + (size_t)b0 * nblk * 9;
    if (KIND == KIND_REMAP) {
      if (p.Bm != 1) {
        q.p.map_x = p.map_x + (size_t)b0 * p.h * p.w;
        q.p.map_y = p.map_y + (size_t)b0 * p.h * p.w;
      }
      if (g.gmap_x) {
        q.gmap_x = g.gmap_x + (size_t)b0 * p.h * p.w;
        q.gmap_y = g.gmap_y + (size_t)b0 * p.h * p.w;
      }
    } else if (p.Bm != 1) {
      q.p.m = p.m + (size_t)b0 * 9;
    }
    const dim3 grid(ceil_div(p.w, GEN_BX), ceil_div(p.h, GEN_BY), q.p.B);
    warp_bwd_generic<T, INTERP, PAD, KIND><<<grid, block, 0, st>>>(q);
  }
  return post_launch("warp_backward");
}

#define KB_DISPATCH_PAD(T, INTERP, KIND, FN, ARG)                                     \
  switch (pad) {                                                                      \
    case KB200_ZEROS: return FN<T, INTERP, KB200_ZEROS, KIND>(ARG, st);               \
    case KB200_BORDER: return FN<T, INTERP, KB200_BORDER, KIND>(ARG, st);             \
    case KB200_REFLECTION: return FN<T, INTERP, KB200_REFLECTION, KIND>(ARG, st);     \
    case KB200_FILL:                                                                  \
      if (KIND == KIND_REMAP) break;                                                  \
      return FN<T, INTERP, KB200_FILL, (KIND == KIND_REMAP ? KIND_AFFINE : KIND)>(ARG, st); \
  }                                                                                   \
  break;

#define KB_DISPATCH_INTERP(T, KIND, FN, ARG)                                       \
  switch (interp) {                                                                \
    case KB200_BILINEAR: KB_DISPATCH_PAD(T, KB200_BILINEAR, KIND, FN, ARG)         \
    case KB200_NEAREST: KB_DISPATCH_PAD(T, KB200_NEAREST, KIND, FN, ARG)           \
    case KB200_BICUBIC: KB_DISPATCH_PAD(T, KB200_BICUBIC, KIND, FN, ARG)           \
  }

template <typename T, int KIND>
static int dispatch_fwd(const WarpParams<T>& p, int interp, int pad, cudaStream_t st) {
  KB_DISPATCH_INTERP(T, KIND, launch_warp_fwd, p)
  set_error("unsupported interp=%d / pad=%d", interp, pad);
  return KB200_EINVAL;
}

template <typename T, int KIND>
static int dispatch_bwd(const WarpGradParams<T>& g, int interp, int pad, cudaStream_t st) {
  KB_DISPATCH_INTERP(T, KIND, launch_warp_bwd, g)
  set_error("unsupported interp=%d / pad=%d", interp, pad);
  return KB200_EINVAL;
}

static int check_common(const void* src, int B, int C, int H, int W, int h, int w, int Bm, int interp, int pad, int dtype,
                        bool allow_fill) {
  KB_CHECK_ARG(src != nullptr, "null src");
  KB_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && h > 0 && w > 0, "non-positive shape B=%d C=%d H=%d W=%d h=%d w=%d", B, C, H, W, h, w);
  KB_CHECK_ARG((long long)H * W < (1ll << 31) && (long long)h * w < (1ll << 31), "plane too large for 32-bit in-plane offsets");
  KB_CHECK_ARG(Bm == B || Bm == 1, "matrix/map batch %d must be %d or 1", Bm, B);
  KB_CHECK_ARG(interp >= KB200_BILINEAR && interp <= KB200_BICUBIC, "bad interp %d", interp);
  KB_CHECK_ARG(pad >= KB200_ZEROS && pad <= (allow_fill ? KB200_FILL : KB200_REFLECTION), "bad pad %d", pad);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  return KB200_OK;
}

template <typename T>
static int warp_forward_t(const void* src, const void* m, const void* bx, const void* by, const void* fill, void* out, int B,
                          int C, int H, int W, int h, int w, int Bm, int projective, int interp, int pad, int align,
                          cudaStream_t st) {
  WarpParams<T> p{};
  p.src = (const T*)src; p.m = (const T*)m; p.bx = (const T*)bx; p.by = (const T*)by;
  p.fill = (const T*)fill; p.out = (T*)out;
  p.B = B; p.C = C; p.H = H; p.W = W; p.h = h; p.w = w; p.Bm = Bm; p.align = align; p.normalized = 0;
  return projective ? dispatch_fwd<T, KIND_PROJ>(p, interp, pad, st) : dispatch_fwd<T, KIND_AFFINE>(p, interp, pad, st);
}

}  // namespace kb200

using namespace kb200;

// The prototypes in include/kornia_b200.h are extern "C"; the definitions below inherit that linkage.

int kb200_abi_version(void) { return KB200_ABI_VERSION; }
const char* kb200_last_error(void) { return g_err; }
const char* kb200_last_warp_variant(void) { return g_variant; }
int kb200_last_warp_launches(void) { return g_warp_launches; }

int kb200_set_option(const char* name, int value) {
  const int i = option_index(name);
  KB_CHECK_ARG(i >= 0, "unknown option '%s'", name ? name : "(null)");
  __atomic_store_n(&g_options[i], value, __ATOMIC_RELAXED);
  return KB200_OK;
}
int kb200_get_option(const char* name) {
  const int i = option_index(name);
  return i < 0 ? (-2147483647 - 1) : option((Option)i);
}

int kb200_warp_forward(const void* src, const void* m, const void* bx, const void* by, const void* fill, void* out, int B,
                       int C, int H, int W, int h, int w, int Bm, int projective, int interp, int pad, int align_corners,
                       int dtype, void* stream) {
  int rc = check_common(src, B, C, H, W, h, w, Bm, interp, pad, dtype, true);
  if (rc) return rc;
  KB_CHECK_ARG(m && bx && by && out, "null pointer argument");
  KB_CHECK_ARG(pad != KB200_FILL || fill, "pad=fill needs a fill vector");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == KB200_F32) {
    // fast path: TMA-staged source tiles (warp_tma.cuh); declines shapes / modes it does not cover.
    // KB200_DISABLE_TMA=1 forces the generic kernel (tests compare the two bit for bit).
    rc = !option(OPT_TMA) ? KB200_EUNSUPPORTED : warp_tma_forward((const float*)src, (const float*)m, (const float*)bx, (const float*)by, (const float*)fill,
                          (float*)out, B, C, H, W, h, w, Bm, projective, interp, pad, align_corners, st);
    if (rc != KB200_EUNSUPPORTED) {
      g_variant = "tma_tile";
      g_warp_launches = warp_tma_last_launches();
      return rc;
    }
    g_variant = "generic";
    g_warp_launches = 1;
    return warp_forward_t<float>(src, m, bx, by, fill, out, B, C, H, W, h, w, Bm, projective, interp, pad, align_corners, st);
  }
  g_variant = "generic";
  g_warp_launches = 1;
  return warp_forward_t<double>(src, m, bx, by, fill, out, B, C, H, W, h, w, Bm, projective, interp, pad, align_corners, st);
}

size_t kb200_warp_backward_workspace_bytes(int B, int h, int w, int dtype) {
  const size_t nblk = (size_t)ceil_div(w, GEN_BX) * ceil_div(h, GEN_BY);
  const size_t generic = (size_t)B * nblk * 9 * (dtype == KB200_F64 ? 8 : 4);
  const size_t tiled = dtype == KB200_F32 ? bwd_tma_workspace_bytes(B, h, w) : 0;
  return generic > tiled ? generic : tiled;
}

template <typename T>
static int warp_backward_t(const void* gout, const void* src, const void* m, const void* bx, const void* by, const void* fill,
                           void* gsrc, void* gm, void* workspace, int B, int C, int H, int W, int h, int w, int Bm,
                           int projective, int interp, int pad, int align, cudaStream_t st) {
  WarpGradParams<T> g{};
  g.p.src = (const T*)src; g.p.m = (const T*)m; g.p.bx = (const T*)bx; g.p.by = (const T*)by; g.p.fill = (const T*)fill;
  g.p.B = B; g.p.C = C; g.p.H = H; g.p.W = W; g.p.h = h; g.p.w = w; g.p.Bm = Bm; g.p.align = align;
  g.gout = (const T*)gout; g.gsrc = (T*)gsrc; g.partial = gm ? (T*)workspace : nullptr;
  g.need_coord_grad = gm != nullptr;
  int rc = projective ? dispatch_bwd<T, KIND_PROJ>(g, interp, pad, st) : dispatch_bwd<T, KIND_AFFINE>(g, interp, pad, st);
  if (rc || !gm) return rc;
  const long long nblk = (long long)ceil_div(w, GEN_BX) * ceil_div(h, GEN_BY);
  warp_gm_reduce<T><<<dim3(9, Bm), 256, 0, st>>>((const T*)workspace, (T*)gm, B, Bm, nblk);
  return post_launch("warp_gm_reduce");
}

int kb200_warp_backward(const void* gout, const void* src, const void* m, const void* bx, const void* by, const void* fill,
                        void* gsrc, void* gm, void* workspace, int B, int C, int H, int W, int h, int w, int Bm,
                        int projective, int interp, int pad, int align_corners, int dtype, void* stream) {
  int rc = check_common(src, B, C, H, W, h, w, Bm, interp, pad, dtype, true);
  if (rc) return rc;
  KB_CHECK_ARG(gout && m && bx && by, "null pointer argument");
  KB_CHECK_ARG(gsrc || gm, "nothing to compute: both gsrc and gm are null");
  KB_CHECK_ARG(!gm || workspace, "gm requested without workspace");
  KB_CHECK_ARG(pad != KB200_FILL || fill, "pad=fill needs a fill vector");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == KB200_F32) {
    rc = warp_tma_backward((const float*)gout, (const float*)src, (const float*)m, (const float*)bx, (const float*)by, (float*)gsrc,
                           (float*)gm, workspace, B, C, H, W, h, w, Bm, projective, interp, pad, align_corners, st);
    if (rc != KB200_EUNSUPPORTED) return rc;
    return warp_backward_t<float>(gout, src, m, bx, by, fill, gsrc, gm, workspace, B, C, H, W, h, w, Bm, projective, interp,
                                  pad, align_corners, st);
  }
  return warp_backward_t<double>(gout, src, m, bx, by, fill, gsrc, gm, workspace, B, C, H, W, h, w, Bm, projective, interp,
                                 pad, align_corners, st);
}

template <typename T>
static int remap_forward_t(const void* src, const void* mx, const void* my, void* out, int B, int C, int H, int W, int h, int w,
                           int Bmap, int normalized, int interp, int pad, int align, cudaStream_t st) {
  WarpParams<T> p{};
  p.src = (const T*)src; p.map_x = (const T*)mx; p.map_y = (const T*)my; p.out = (T*)out;
  p.B = B; p.C = C; p.H = H; p.W = W; p.h = h; p.w = w; p.Bm = Bmap; p.align = align; p.normalized = normalized;
  return dispatch_fwd<T, KIND_REMAP>(p, interp, pad, st);
}

int kb200_remap_forward(const void* src, const void* map_x, const void* map_y, void* out, int B, int C, int H, int W, int h,
                        int w, int Bmap, int normalized, int interp, int pad, int align_corners, int dtype, void* stream) {
  int rc = check_common(src, B, C, H, W, h, w, Bmap, interp, pad, dtype, false);
  if (rc) return rc;
  KB_CHECK_ARG(map_x && map_y && out, "null pointer argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == KB200_F32) {
    rc = remap_tiled_forward((const float*)src, (const float*)map_x, (const float*)map_y, (float*)out, B, C, H, W, h, w, Bmap, normalized,
                             interp, pad, align_corners, st);
    if (rc != KB200_EUNSUPPORTED) return rc;
    return remap_forward_t<float>(src, map_x, map_y, out, B, C, H, W, h, w, Bmap, normalized, interp, pad, align_corners, st);
  }
  return remap_forward_t<double>(src, map_x, map_y, out, B, C, H, W, h, w, Bmap, normalized, interp, pad, align_corners, st);
}

int kb200_undistort_forward(const void* src, const void* lens, void* out, int B, int C, int H, int W, int dtype, void* stream) {
  KB_CHECK_ARG(src && lens && out, "null pointer argument");
  KB_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0, "non-positive shape");
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  int rc = KB200_EUNSUPPORTED;
  if (dtype == KB200_F32) {
    rc = undistort_tiled_forward((const float*)src, (const float*)lens, (float*)out, B, C, H, W, (cudaStream_t)stream);
  }
  if (rc == KB200_EUNSUPPORTED) set_error("the fused undistort kernel covers fp32 images of 1 or 3 channels with a width divisible by 4");
  return rc;
}

template <typename T>
static int remap_backward_t(const void* gout, const void* src, const void* mx, const void* my, void* gsrc, void* gmx, void* gmy,
                            int B, int C, int H, int W, int h, int w, int Bmap, int normalized, int interp, int pad, int align,
                            cudaStream_t st) {
  WarpGradParams<T> g{};
  g.p.src = (const T*)src; g.p.map_x = (const T*)mx; g.p.map_y = (const T*)my;
  g.p.B = B; g.p.C = C; g.p.H = H; g.p.W = W; g.p.h = h; g.p.w = w; g.p.Bm = Bmap; g.p.align = align;
  g.p.normalized = normalized;
  g.gout = (const T*)gout; g.gsrc = (T*)gsrc; g.gmap_x = (T*)gmx; g.gmap_y = (T*)gmy;
  g.need_coord_grad = gmx != nullptr;
  return dispatch_bwd<T, KIND_REMAP>(g, interp, pad, st);
}

int kb200_remap_backward(const void* gout, const void* src, const void* map_x, const void* map_y, void* gsrc, void* gmap_x,
                         void* gmap_y, int B, int C, int H, int W, int h, int w, int Bmap, int normalized, int interp, int pad,
                         int align_corners, int dtype, void* stream) {
  int rc = check_common(src, B, C, H, W, h, w, Bmap, interp, pad, dtype, false);
  if (rc) return rc;
  KB_CHECK_ARG(gout && map_x && map_y, "null pointer argument");
  KB_CHECK_ARG((gmap_x == nullptr) == (gmap_y == nullptr), "gmap_x and gmap_y must be given together");
  KB_CHECK_ARG(gsrc || gmap_x, "nothing to compute");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == KB200_F32)
    return remap_backward_t<float>(gout, src, map_x, map_y, gsrc, gmap_x, gmap_y, B, C, H, W, h, w, Bmap, normalized, interp, pad,
                                   align_corners, st);
  return remap_backward_t<double>(gout, src, map_x, map_y, gsrc, gmap_x, gmap_y, B, C, H, W, h, w, Bmap, normalized, interp, pad,
                                  align_corners, st);
}

// ------------------------------------------------------------------------------------------
// filters
// ------------------------------------------------------------------------------------------
static int check_filter(const void* x, const void* k, int B, int C, int H, int W, int Bk, int kh, int kw, int border, int same,
                        int dtype) {
  KB_CHECK_ARG(x && k, "null pointer argument");
  KB_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && Bk > 0 && kh > 0 && kw > 0, "non-positive shape");
  KB_CHECK_ARG(B % Bk == 0, "kernel batch %d must divide the input batch %d", Bk, B);
  KB_CHECK_ARG((long long)H * W < (1ll << 31), "plane too large");
  KB_CHECK_ARG(border >= KB200_CONSTANT && border <= KB200_CIRCULAR, "bad border %d", border);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (same) {
    const int ph = kh - 1 - (kh - 1) / 2, pw = kw - 1 - (kw - 1) / 2;  // the larger (rear) pad
    if (border == KB200_REFLECT) KB_CHECK_ARG(ph < H && pw < W, "reflect padding (%d,%d) must be smaller than the image (%d,%d)", ph, pw, H, W);
    if (border == KB200_CIRCULAR) KB_CHECK_ARG(ph <= H && pw <= W, "circular padding (%d,%d) must not exceed the image (%d,%d)", ph, pw, H, W);
  } else {
    KB_CHECK_ARG(kh <= H && kw <= W, "'valid' needs kernel (%d,%d) <= image (%d,%d)", kh, kw, H, W);
  }
  return KB200_OK;
}

template <typename T>
static FilterParams<T> make_fp(const void* x, const void* k, void* out, int B, int C, int H, int W, int Bk, int kh, int kw,
                               int same) {
  FilterParams<T> p{};
  p.x = (const T*)x; p.k = (const T*)k; p.out = (T*)out;
  p.B = B; p.C = C; p.H = H; p.W = W; p.Bk = Bk; p.kh = kh; p.kw = kw;
  p.top = same ? (kh - 1) / 2 : 0;
  p.left = same ? (kw - 1) / 2 : 0;
  p.Ho = same ? H : H - kh + 1;
  p.Wo = same ? W : W - kw + 1;
  return p;
}

#define KB_BORDER_SWITCH(border, same, ...)                   \
  switch ((same) ? (border) : KB200_CONSTANT) {                \
    case KB200_CONSTANT: { constexpr int BD = KB200_CONSTANT; __VA_ARGS__; break; }   \
    case KB200_REFLECT: { constexpr int BD = KB200_REFLECT; __VA_ARGS__; break; }     \
    case KB200_REPLICATE: { constexpr int BD = KB200_REPLICATE; __VA_ARGS__; break; } \
    case KB200_CIRCULAR: { constexpr int BD = KB200_CIRCULAR; __VA_ARGS__; break; }   \
  }

template <typename T>
static int filter2d_forward_t(const void* x, const void* k, void* out, int B, int C, int H, int W, int Bk, int kh, int kw,
                              int border, int same, cudaStream_t st) {
  FilterParams<T> p = make_fp<T>(x, k, out, B, C, H, W, Bk, kh, kw, same);
  const dim3 grid(ceil_div(p.Wo, 32), ceil_div(p.Ho, 8), B * C);
  KB_BORDER_SWITCH(border, same, (filter2d_fwd_generic<T, BD><<<grid, dim3(32, 8), 0, st>>>(p)));
  return post_launch("filter2d_forward");
}

int kb200_filter2d_forward(const void* x, const void* kernel, void* out, int B, int C, int H, int W, int Bk, int kh, int kw,
                           int border, int same, int dtype, void* stream) {
  int rc = check_filter(x, kernel, B, C, H, W, Bk, kh, kw, border, same, dtype);
  if (rc) return rc;
  KB_CHECK_ARG(out, "null out");
  KB_CHECK_ARG((long long)B * C <= MAX_Z, "B*C = %lld planes exceed the %d-plane launch limit", (long long)B * C, MAX_Z);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == KB200_F32) {
    rc = filter2d_tiled_forward((const float*)x, (const float*)kernel, (float*)out, B, C, H, W, Bk, kh, kw, border, same, st);  // K in {3, 5, 7}
    if (rc != KB200_EUNSUPPORTED) return rc;
    rc = filter2d_taps_forward((const float*)x, (const float*)kernel, (float*)out, B, C, H, W, Bk, kh, kw, border, same, st);  // odd K 9..31
    if (rc != KB200_EUNSUPPORTED) return rc;
    return filter2d_forward_t<float>(x, kernel, out, B, C, H, W, Bk, kh, kw, border, same, st);
  }
  return filter2d_forward_t<double>(x, kernel, out, B, C, H, W, Bk, kh, kw, border, same, st);
}

int kb200_pyrdown_forward(const void* x, const void* kernel, void* out, int B, int C, int H, int W, int Bk, int border, int dtype,
                          void* stream) {
  int rc = check_filter(x, kernel, B, C, H, W, Bk, 5, 5, border, 1, dtype);
  if (rc) return rc;
  KB_CHECK_ARG(out, "null out");
  if (dtype != KB200_F32) {
    set_error("the fused pyrdown kernel is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  rc = pyrdown_tiled_forward((const float*)x, (const float*)kernel, (float*)out, B, C, H, W, Bk, border, (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED) set_error("the fused pyrdown kernel needs an even height, a width divisible by 4 and a non-circular border");
  return rc;
}

template <typename T>
static int filter2d_backward_input_t(const void* gout, const void* k, void* gx, int B, int C, int H, int W, int Bk, int kh,
                                     int kw, int border, int same, cudaStream_t st) {
  FilterParams<T> p = make_fp<T>(nullptr, k, nullptr, B, C, H, W, Bk, kh, kw, same);
  const int bottom = same ? (kh - 1) - p.top : 0, right = same ? (kw - 1) - p.left : 0;
  const dim3 grid(ceil_div(W, 32), ceil_div(H, 8), B * C);
  KB_BORDER_SWITCH(border, same,
                   (filter2d_bwd_input_generic<T, BD><<<grid, dim3(32, 8), 0, st>>>(p, (const T*)gout, (T*)gx, bottom, right)));
  return post_launch("filter2d_backward_input");
}

int kb200_filter2d_backward_input(const void* gout, const void* kernel, void* gx, int B, int C, int H, int W, int Bk, int kh,
                                  int kw, int border, int same, int dtype, void* stream) {
  int rc = check_filter(gout, kernel, B, C, H, W, Bk, kh, kw, border, same, dtype);
  if (rc) return rc;
  KB_CHECK_ARG(gx, "null gx");
  KB_CHECK_ARG((long long)B * C <= MAX_Z, "B*C = %lld planes exceed the %d-plane launch limit", (long long)B * C, MAX_Z);
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == KB200_F32 ? filter2d_backward_input_t<float>(gout, kernel, gx, B, C, H, W, Bk, kh, kw, border, same, st)
                            : filter2d_backward_input_t<double>(gout, kernel, gx, B, C, H, W, Bk, kh, kw, border, same, st);
}

size_t kb200_filter2d_backward_kernel_workspace_bytes(int B, int C, int H, int W, int Bk, int kh, int kw, int dtype) {
  (void)H; (void)W; (void)Bk;
  return (size_t)B * C * kh * kw * (dtype == KB200_F64 ? 8 : 4);
}

template <typename T>
static int filter2d_backward_kernel_t(const void* gout, const void* x, void* gk, void* ws, int B, int C, int H, int W, int Bk,
                                      int kh, int kw, int border, int same, cudaStream_t st) {
  FilterParams<T> p = make_fp<T>(x, nullptr, nullptr, B, C, H, W, Bk, kh, kw, same);
  const dim3 grid(kh * kw, B * C);
  KB_BORDER_SWITCH(border, same, (filter2d_bwd_kernel_stage1<T, BD><<<grid, 256, 0, st>>>(p, (const T*)gout, (T*)ws)));
  int rc = post_launch("filter2d_backward_kernel stage1");
  if (rc) return rc;
  const int taps = kh * kw;
  filter2d_bwd_kernel_stage2<T><<<dim3(ceil_div(taps, 128), Bk), 128, 0, st>>>((const T*)ws, (T*)gk, B, C, Bk, taps);
  return post_launch("filter2d_backward_kernel stage2");
}

int kb200_filter2d_backward_kernel(const void* gout, const void* x, void* gkernel, void* workspace, int B, int C, int H, int W,
                                   int Bk, int kh, int kw, int border, int same, int dtype, void* stream) {
  int rc = check_filter(x, gout, B, C, H, W, Bk, kh, kw, border, same, dtype);
  if (rc) return rc;
  KB_CHECK_ARG(gkernel && workspace, "null gkernel / workspace");
  KB_CHECK_ARG((long long)B * C <= MAX_Z && kh * kw <= 65535 * 32, "launch limits exceeded");
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == KB200_F32
             ? filter2d_backward_kernel_t<float>(gout, x, gkernel, workspace, B, C, H, W, Bk, kh, kw, border, same, st)
             : filter2d_backward_kernel_t<double>(gout, x, gkernel, workspace, B, C, H, W, Bk, kh, kw, border, same, st);
}

template <typename T>
static int sepfilter_forward_t(const void* x, const void* kx, const void* ky, void* out, int B, int C, int H, int W, int Bkx,
                               int kw, int Bky, int kh, int border, int same, cudaStream_t st) {
  SepParams<T> p{};
  p.x = (const T*)x; p.kx = (const T*)kx; p.ky = (const T*)ky; p.out = (T*)out;
  p.B = B; p.C = C; p.H = H; p.W = W; p.Bkx = Bkx; p.kw = kw; p.Bky = Bky; p.kh = kh;
  p.top = same ? (kh - 1) / 2 : 0;
  p.left = same ? (kw - 1) / 2 : 0;
  p.Ho = same ? H : H - kh + 1;
  p.Wo = same ? W : W - kw + 1;
  const int in_w = SEP_TW + kw - 1, in_h = SEP_TH + kh - 1;
  const size_t smem = ((size_t)in_h * in_w + (size_t)in_h * SEP_TW + kw + kh) * sizeof(T);
  if (smem > 200 * 1024) {
    set_error("separable kernel (%d,%d) needs %zu B of shared memory; use two filter2d passes", kh, kw, smem);
    return KB200_EUNSUPPORTED;
  }
  const dim3 grid(ceil_div(p.Wo, SEP_TW), ceil_div(p.Ho, SEP_TH), B * C);
  KB_BORDER_SWITCH(border, same, {
    auto kern = sepfilter_fwd_generic<T, BD>;
    KB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, 256, smem, st>>>(p);
  });
  return post_launch("sepfilter_forward");
}

int kb200_sepfilter_forward(const void* x, const void* kernel_x, const void* kernel_y, void* out, int B, int C, int H, int W,
                            int Bkx, int kw, int Bky, int kh, int border, int same, int dtype, void* stream) {
  int rc = check_filter(x, kernel_x, B, C, H, W, Bkx, kh, kw, border, same, dtype);
  if (rc) return rc;
  KB_CHECK_ARG(kernel_y && out, "null pointer argument");
  KB_CHECK_ARG(Bky > 0 && B % Bky == 0, "kernel_y batch %d must divide the input batch %d", Bky, B);
  KB_CHECK_ARG((long long)B * C <= MAX_Z, "B*C = %lld planes exceed the %d-plane launch limit", (long long)B * C, MAX_Z);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == KB200_F32) {
    rc = sepfilter_tiled_forward((const float*)x, (const float*)kernel_x, (const float*)kernel_y, (float*)out, B, C, H, W, Bkx,
                                 kw, Bky, kh, border, same, st);
    if (rc != KB200_EUNSUPPORTED) return rc;
    return sepfilter_forward_t<float>(x, kernel_x, kernel_y, out, B, C, H, W, Bkx, kw, Bky, kh, border, same, st);
  }
  return sepfilter_forward_t<double>(x, kernel_x, kernel_y, out, B, C, H, W, Bkx, kw, Bky, kh, border, same, st);
}


int kb200_perspective_from_points(const void* points_src, const void* points_dst, void* H_out, int B, int dtype, int variant,
                                  void* stream) {
  KB_CHECK_ARG(points_src && points_dst && H_out && B > 0, "bad arguments");
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(B, 128);
  if (dtype == KB200_F32)
    perspective_from_points_kernel<float><<<grid, 128, 0, st>>>((const float*)points_src, (const float*)points_dst, (float*)H_out, B,
                                                               variant);
  else
    perspective_from_points_kernel<double><<<grid, 128, 0, st>>>((const double*)points_src, (const double*)points_dst,
                                                                (double*)H_out, B, variant);
  return post_launch("perspective_from_points");
}

int kb200_ssim_forward(const void* img1, const void* img2, const void* taps, void* out, int planes, int H, int W, int K, double C1,
                       double C2, double eps, int dtype, void* stream) {
  KB_CHECK_ARG(img1 && img2 && taps && out, "null pointer argument");
  KB_CHECK_ARG(planes > 0 && H > 0 && W > 0 && K > 0, "bad sizes planes=%d H=%d W=%d K=%d", planes, H, W, K);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused SSIM kernel is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  KB_CHECK_ARG(K % 2 == 0 || K > SSIM_MAX_K || (K / 2 < H && K / 2 < W), "reflect border of %d needs an image larger than %d x %d", K / 2, H, W);
  const int rc = ssim_vwalk_forward((const float*)img1, (const float*)img2, (const float*)taps, (float*)out, planes, H, W, K, (float)C1,
                                    (float)C2, (float)eps, (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED)
    set_error("the fused SSIM kernel handles odd windows up to %d taps on rows that are a multiple of 4 floats (16-byte aligned), got K=%d W=%d",
              SSIM_MAX_K, K, W);
  return rc;
}

int kb200_rotation_matrix2d(const void* center, const void* angle, const void* scale, void* M_out, int B, int dtype, int variant,
                            void* stream) {
  KB_CHECK_ARG(center && angle && scale && M_out && B > 0, "bad arguments");
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(B, 128);
  if (dtype == KB200_F32)
    rotation_matrix2d_kernel<float><<<grid, 128, 0, st>>>((const float*)center, (const float*)angle, (const float*)scale, (float*)M_out, B,
                                                         variant);
  else
    rotation_matrix2d_kernel<double><<<grid, 128, 0, st>>>((const double*)center, (const double*)angle, (const double*)scale,
                                                          (double*)M_out, B, variant);
  return post_launch("rotation_matrix2d");
}

int kb200_spatial_gradient_forward(const void* x, const double* taps, void* out, int planes, int H, int W, int nout, int k,
                                   int magnitude, double eps, int dtype, void* stream) {
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  return spatial_gradient_forward(x, taps, out, planes, H, W, nout, k, magnitude, eps, dtype, (cudaStream_t)stream);
}

int kb200_spatial_gradient_backward(const void* gout, const double* taps, void* gx, int planes, int H, int W, int nout, int k,
                                    int dtype, void* stream) {
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  return spatial_gradient_backward(gout, taps, gx, planes, H, W, nout, k, dtype, (cudaStream_t)stream);
}

int kb200_feature_response_forward(const void* x, const double* stencil, const void* blur_taps, double k, const void* k_ptr, const void* s4,
                                   void* out, int planes, int C, int H, int W, int stencil_k, int blur_k, int kind, int dtype, void* stream) {
  KB_CHECK_ARG(x && stencil && out, "null pointer argument");
  KB_CHECK_ARG(kind == RESP_HARRIS || kind == RESP_GFTT || kind == RESP_HESSIAN, "bad response kind %d", kind);
  KB_CHECK_ARG(planes > 0 && H > 0 && W > 0 && C > 0 && planes % C == 0, "bad sizes planes=%d C=%d H=%d W=%d", planes, C, H, W);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  const bool corner = kind != RESP_HESSIAN;
  KB_CHECK_ARG(!corner || blur_taps, "null blur taps");
  KB_CHECK_ARG(!corner || blur_k != CORNER_K || (CORNER_K / 2 < H && CORNER_K / 2 < W), "reflect border of %d needs an image larger than %d x %d",
               CORNER_K / 2, H, W);
  if (dtype != KB200_F32 || (corner ? stencil_k != 3 || blur_k != CORNER_K : stencil_k != 3 && stencil_k != 5)) {
    set_error("the fused response kernels are fp32 only, with 3x3 stencils and a %d-tap blur (Harris, GFTT) or 3x3 / 5x5 stencils (Hessian)",
              CORNER_K);
    return KB200_EUNSUPPORTED;
  }
  const int rc = corner ? corner_vwalk_forward((const float*)x, stencil, (const float*)blur_taps, (float)k, (const float*)k_ptr, (const float*)s4,
                                               (float*)out, planes, C, H, W, kind, (cudaStream_t)stream)
                        : hessian_tiled_forward((const float*)x, stencil, (const float*)s4, (float*)out, planes, C, H, W, stencil_k,
                                                (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED)
    set_error("the fused response kernels need rows that are a multiple of 4 floats (16-byte aligned) and an image larger than the stencil, "
              "got H=%d W=%d", H, W);
  return rc;
}

int kb200_scale_octave_forward(const void* x, const double* taps, const int* ksizes, int L, void* out, int planes, int H, int W, int dtype,
                               void* stream) {
  KB_CHECK_ARG(x && taps && ksizes && out, "null pointer argument");
  KB_CHECK_ARG(planes > 0 && H > 0 && W > 0 && L > 0, "bad sizes planes=%d L=%d H=%d W=%d", planes, L, H, W);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  for (int l = 0; l < L; ++l) KB_CHECK_ARG(ksizes[l] >= (l == 0 ? 0 : 1), "bad tap count %d of level %d", ksizes[l], l);
  const int rc = dtype == KB200_F32 ? octave_vwalk_forward((const float*)x, taps, ksizes, L, (float*)out, planes, H, W, (cudaStream_t)stream)
                                    : KB200_EUNSUPPORTED;
  if (rc == KB200_EUNSUPPORTED)
    set_error("the fused octave kernel is fp32 only, for the instantiated tap chains, with every tap count <= min(H, W) and rows that are a "
              "multiple of 4 floats (16-byte aligned), got L=%d H=%d W=%d", L, H, W);
  return rc;
}

int kb200_nms2d_forward(const void* x, void* out, int B, int C, int H, int W, long long sB, long long sC, int k, int values, int dtype,
                        void* stream) {
  KB_CHECK_ARG(x && out, "null pointer argument");
  KB_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0, "bad sizes B=%d C=%d H=%d W=%d", B, C, H, W);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  const int rc = dtype == KB200_F32 ? nms2d_forward((const float*)x, out, B, C, H, W, sB, sC, k, values != 0, (cudaStream_t)stream)
                                    : KB200_EUNSUPPORTED;
  if (rc == KB200_EUNSUPPORTED)
    set_error("the fused 2-D non-maximum suppression is fp32 only, for square odd kernel sizes 3..31, got k=%d", k);
  return rc;
}

int kb200_nms3d_forward(const void* x, void* out0, void* out1, int B, int C, int L, int H, int W, long long sB, long long sC,
                        long long sL, int mode, int dtype, void* stream) {
  KB_CHECK_ARG(x && out0 && (mode != 2 || out1), "null pointer argument");
  KB_CHECK_ARG(B > 0 && C > 0 && L > 0 && H > 0 && W > 0, "bad sizes B=%d C=%d L=%d H=%d W=%d", B, C, L, H, W);
  KB_CHECK_ARG(mode >= 0 && mode <= 2, "bad mode %d", mode);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  const int rc = dtype == KB200_F32 ? nms3d_forward((const float*)x, out0, out1, B, C, L, H, W, sB, sC, sL, mode, (cudaStream_t)stream)
                                    : KB200_EUNSUPPORTED;
  if (rc == KB200_EUNSUPPORTED) set_error("the fused 3-D non-maximum suppression is fp32 only");
  return rc;
}

int kb200_quad_interp3d_forward(const void* x, const void* mask, void* coords, void* y, int B, int C, int L, int H, int W, long long sB,
                                long long sC, long long sL, long long ysB, long long ysC, long long ysL, long long ysH,
                                long long ysW, int n_iters, int radius, float max_shift, float bonus, int add_bonus, int allow_scale,
                                int dtype, void* stream) {
  KB_CHECK_ARG(x && coords && y, "null pointer argument");
  KB_CHECK_ARG(B > 0 && C > 0 && L > 0 && H > 0 && W > 0, "bad sizes B=%d C=%d L=%d H=%d W=%d", B, C, L, H, W);
  KB_CHECK_ARG(radius >= 0, "bad dilation radius %d", radius);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused sub-pixel refinement is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  return quad_interp3d_forward((const float*)x, (const unsigned char*)mask, (float*)coords, (float*)y, B, C, L, H, W, sB, sC, sL, ysB,
                               ysC, ysL, ysH, ysW, n_iters, radius, max_shift, bonus, add_bonus, allow_scale, (cudaStream_t)stream);
}

namespace kb200 {
// siftdesc.cu / patch_orientation.cu (their kernels are not templates, so their headers are included there only)
int sift_describe_forward(const float* x, const float* gk, const float* pk, float* out, long long N, int P, long long sB, long long sH, int A,
                          int S, int K, int stride, int pad, int rootsift, float clipval, float eps, cudaStream_t st);
int patch_orientation_forward(const float* x, const float* weighting, const float* smooth, float* out, long long N, int P, long long sB,
                              long long sH, int A, float eps, cudaStream_t st);
}  // namespace kb200

int kb200_sift_describe_forward(const void* x, const void* gk, const void* pk, void* out, long long N, int P, long long sB, long long sH,
                                int num_ang_bins, int num_spatial_bins, int ksize, int stride, int pad, int rootsift, float clipval,
                                float eps, int dtype, void* stream) {
  KB_CHECK_ARG(N >= 0 && P > 0 && num_ang_bins > 0 && num_spatial_bins > 0 && ksize > 0 && stride > 0 && pad >= 0,
               "bad sizes N=%lld P=%d A=%d S=%d K=%d stride=%d pad=%d", N, P, num_ang_bins, num_spatial_bins, ksize, stride, pad);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused SIFT descriptor is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  if (N == 0) return KB200_OK;
  KB_CHECK_ARG(x && gk && pk && out, "null pointer argument");
  const int rc = sift_describe_forward((const float*)x, (const float*)gk, (const float*)pk, (float*)out, N, P, sB, sH, num_ang_bins,
                                       num_spatial_bins, ksize, stride, pad, rootsift, clipval, eps, (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED) set_error("SIFT configuration P=%d A=%d S=%d is outside the fused kernel's envelope", P, num_ang_bins, num_spatial_bins);
  return rc;
}

int kb200_patch_orientation_forward(const void* x, const void* weighting, const void* smooth, void* out, long long N, int P, long long sB,
                                    long long sH, int num_ang_bins, float eps, int dtype, void* stream) {
  KB_CHECK_ARG(N >= 0 && P > 0 && num_ang_bins > 0, "bad sizes N=%lld P=%d A=%d", N, P, num_ang_bins);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused dominant-orientation estimate is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  if (N == 0) return KB200_OK;
  KB_CHECK_ARG(x && weighting && smooth && out, "null pointer argument");
  const int rc = patch_orientation_forward((const float*)x, (const float*)weighting, (const float*)smooth, (float*)out, N, P, sB, sH,
                                           num_ang_bins, eps, (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED) set_error("orientation configuration P=%d A=%d is outside the fused kernel's envelope", P, num_ang_bins);
  return rc;
}

namespace kb200 {
// laf_patches.cu (its kernel is not a template, so its header is included there only)
int extract_patches_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                            void* out, long long B, long long N, int C, int PS, int normalize, int select_level, cudaStream_t st);
}  // namespace kb200

int kb200_extract_patches_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                                  void* out, long long B, long long N, int C, int PS, int normalize, int select_level, int dtype,
                                  void* stream) {
  KB_CHECK_ARG(B >= 0 && N >= 0 && C > 0 && PS > 0, "bad sizes B=%lld N=%lld C=%d PS=%d", B, N, C, PS);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused patch extraction is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  return extract_patches_forward(levels, level_dims, n_levels, laf, base, out, B, N, C, PS, normalize, select_level, (cudaStream_t)stream);
}

namespace kb200 {
// affine_shape.cu (its kernels are not templates, so its header is included there only)
int patch_affine_shape_forward(const float* x, const float* weighting, float* out, long long N, int P, long long sB, long long sH, float eps,
                               cudaStream_t st);
int laf_affine_shape_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                             const void* weighting, void* out, long long B, long long N, int PS, float eps, int preserve_orientation,
                             cudaStream_t st);
}  // namespace kb200

int kb200_patch_affine_shape_forward(const void* x, const void* weighting, void* out, long long N, int P, long long sB, long long sH, float eps,
                                     int dtype, void* stream) {
  KB_CHECK_ARG(N >= 0 && P > 0, "bad sizes N=%lld P=%d", N, P);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused affine shape estimate is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  if (N == 0) return KB200_OK;
  KB_CHECK_ARG(x && weighting && out, "null pointer argument");
  const int rc = patch_affine_shape_forward((const float*)x, (const float*)weighting, (float*)out, N, P, sB, sH, eps, (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED) set_error("patch size %d is outside the fused affine shape kernel's envelope", P);
  return rc;
}

int kb200_laf_affine_shape_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                                   const void* weighting, void* out, long long B, long long N, int PS, float eps, int preserve_orientation,
                                   int dtype, void* stream) {
  KB_CHECK_ARG(B >= 0 && N >= 0 && PS > 0, "bad sizes B=%lld N=%lld PS=%d", B, N, PS);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  if (dtype != KB200_F32) {
    set_error("the fused LAF affine shape estimate is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  const int rc = laf_affine_shape_forward(levels, level_dims, n_levels, laf, base, weighting, out, B, N, PS, eps, preserve_orientation,
                                          (cudaStream_t)stream);
  if (rc == KB200_EUNSUPPORTED) set_error("patch size %d is outside the fused affine shape kernel's envelope", PS);
  return rc;
}

int kb200_sepfilter_lerp_forward(const void* x, const void* kernel_x, const void* kernel_y, void* out, int B, int C, int H, int W,
                                 int Bkx, int kw, int Bky, int kh, int border, int same, double weight, int dtype, void* stream) {
  int rc = check_filter(x, kernel_x, B, C, H, W, Bkx, kh, kw, border, same, dtype);
  if (rc) return rc;
  KB_CHECK_ARG(kernel_y && out, "null pointer argument");
  KB_CHECK_ARG(Bky > 0 && B % Bky == 0, "kernel_y batch %d must divide the input batch %d", Bky, B);
  if (dtype != KB200_F32 || (long long)B * C > MAX_Z) {
    set_error("the fused filter + lerp kernel is fp32 only");
    return KB200_EUNSUPPORTED;
  }
  const float w = (float)weight;
  rc = sepfilter_tiled_forward((const float*)x, (const float*)kernel_x, (const float*)kernel_y, (float*)out, B, C, H, W, Bkx, kw, Bky,
                               kh, border, same, (cudaStream_t)stream, &w);
  if (rc == KB200_EUNSUPPORTED) set_error("the fused filter + lerp kernel covers square odd kernels up to 11 taps, 'same', non-circular borders");
  return rc;
}

int kb200_warp_prelude(const void* M, void* m_out, int B, int rows, int H, int W, int h, int w, int dtype, int variant,
                       void* stream) {
  KB_CHECK_ARG(M && m_out && B > 0, "bad arguments");
  KB_CHECK_ARG(rows == 2 || rows == 3, "rows must be 2 (affine) or 3 (projective), got %d", rows);
  KB_CHECK_ARG(H > 0 && W > 0 && h > 0 && w > 0, "non-positive size");
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  // normal_transform_pixel (conversions.py:1753-1765): python floats -> fp32 tensor -> cast to M's dtype
  const float sx_s = (float)(2.0 / (W == 1 ? 1e-14 : (double)W - 1.0)), sy_s = (float)(2.0 / (H == 1 ? 1e-14 : (double)H - 1.0));
  const float sx_d = (float)(2.0 / (w == 1 ? 1e-14 : (double)w - 1.0)), sy_d = (float)(2.0 / (h == 1 ? 1e-14 : (double)h - 1.0));
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(B, 128);
  if (dtype == KB200_F32)
    warp_prelude_kernel<float><<<grid, 128, 0, st>>>((const float*)M, (float*)m_out, B, rows, sx_s, sy_s, sx_d, sy_d, variant);
  else
    warp_prelude_kernel<double><<<grid, 128, 0, st>>>((const double*)M, (double*)m_out, B, rows, sx_s, sy_s, sx_d, sy_d, variant);
  return post_launch("warp_prelude");
}

int kb200_warp_prelude_backward(const void* m, const void* gm, void* gM, int B, int rows, int H, int W, int h, int w, int dtype,
                                void* stream) {
  KB_CHECK_ARG(m && gm && gM && B > 0, "bad arguments");
  KB_CHECK_ARG(rows == 2 || rows == 3, "rows must be 2 (affine) or 3 (projective), got %d", rows);
  KB_CHECK_ARG(dtype == KB200_F32 || dtype == KB200_F64, "bad dtype %d", dtype);
  const float sx_s = (float)(2.0 / (W == 1 ? 1e-14 : (double)W - 1.0)), sy_s = (float)(2.0 / (H == 1 ? 1e-14 : (double)H - 1.0));
  const float sx_d = (float)(2.0 / (w == 1 ? 1e-14 : (double)w - 1.0)), sy_d = (float)(2.0 / (h == 1 ? 1e-14 : (double)h - 1.0));
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ceil_div(B, 128);
  if (dtype == KB200_F32)
    warp_prelude_backward_kernel<float><<<grid, 128, 0, st>>>((const float*)m, (const float*)gm, (float*)gM, B, rows, sx_s, sy_s, sx_d, sy_d);
  else
    warp_prelude_backward_kernel<double><<<grid, 128, 0, st>>>((const double*)m, (const double*)gm, (double*)gM, B, rows, sx_s, sy_s, sx_d,
                                                               sy_d);
  return post_launch("warp_prelude_backward");
}

// ------------------------------------------------------------------------------------------
// diagnostics
// ------------------------------------------------------------------------------------------
namespace kb200 {
__global__ void fastdiv_check_kernel(const float* __restrict__ num, const float* __restrict__ den, int n, int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float a = num[i], b = den[i];
  if (!(fabsf(b) >= 8.67361738e-19f)) return;  // outside the window the kernel uses __fdiv_rn itself
  const float q = div_by_rcp(a, b, refined_rcp(b));
  const float want = __fdiv_rn(a, b);
  // NaN == NaN for this purpose; differing non-finite / sub-2^-24 results cannot change a sampled pixel
  const bool same = (__float_as_uint(q) == __float_as_uint(want)) || (q != q && want != want) ||
                    (!(fabsf(want) <= 3.0e38f) && !(fabsf(q) <= 3.0e38f)) || (fabsf(want) < 5.9e-8f && fabsf(q) < 5.9e-8f);
  if (!same) atomicAdd(bad, 1);
}
}  // namespace kb200

int kb200_debug_fastdiv_mismatches(const float* num, const float* den, int n, int* count, void* stream) {
  KB_CHECK_ARG(num && den && count && n > 0, "bad arguments");
  fastdiv_check_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(num, den, n, count);
  return post_launch("fastdiv_check");
}
