// kornia_b200 -- non-maximum suppression (kornia/geometry/subpix/nms.py) in one pass per call (fp32).
//
// nms2d / NonMaximaSuppression2d for a square odd K = 3 .. 31, and nms3d (3, 3, 3) / nms3d_minmax.  Every form keeps a
// position when x > M, M the NaN-propagating maximum of a neighbour set (for the minima of nms3d_minmax: x < the
// NaN-propagating minimum), so a NaN anywhere in the set, or at the centre, gives False:
//  * K = 3, 5, 7 (the reference's explicit comparisons): the K*K - 1 neighbours; the outer (K - 1) / 2 ring is False.
//  * K >= 9 (the reference's one-hot F.conv2d of the replicate-padded image): the K*K - 1 replicate-clamped neighbours
//    and 0 (the all-zero centre channel).  A window, centre included, that holds a non-finite texel is False: 0 * Inf and
//    0 * NaN make every channel NaN.  Texels are staged as NaN when they are not finite, which gives both rules.
//  * 3-D: the 26 neighbours; the border levels, rows and columns are False.
// The values form writes x * keep as a real multiply, as the composition does: a masked-off negative gives -0, a
// masked-off NaN or +-Inf gives NaN.  (A staged NaN of the K >= 9 form times 0 is the same canonical NaN as the
// non-finite texel it stands for times 0.)  max.NaN / min.NaN and the comparisons do not flush subnormals.
//
// 2-D: persistent CTAs over 64 x 32 tiles.  A CTA stages its tile plus a (K - 1) / 2 halo, replicate-clamped, in shared
// memory; takes for every staged row the K-column maximum (and on the tile's own rows the maximum without the centre
// column); then per output the maximum of those down its K rows: 2K - 2 max per output rather than K*K - 1.
// 3-D: persistent CTAs over 128 x 8 tiles of one (b, c) volume walk the L axis.  Per level the tile plus a one-texel halo
// is staged, each thread reduces the 3 x 3 max and min of its 4 columns, and a three-level register ring gives level
// l - 1 its 26-neighbour max / min once level l is staged, so each level is read once per tile.
//
// The source's H x W planes are dense; the b, c (and 3-D: level) strides are arguments, so a permuted view is read in
// place.  Outputs are contiguous; 4-column groups are stored as uchar4 / float4 where aligned.
//
// Launched by nms.cu; tests/test_nms_gpu.py checks both kernels bit for bit against the composition, and tools/hostemu
// (run_emu --nms) runs them on the host against a scalar restatement.
#pragma once
#include "common.cuh"

namespace kb200 {

constexpr int NMS_TW = 64, NMS_TH = 32, NMS_NT = 256;     // 2-D tile; 16 x 16 threads of 4 columns x 2 rows
constexpr int NMS3_TW = 128, NMS3_TH = 8, NMS3_NT = 256;  // 3-D tile; 32 x 8 threads of 4 columns x 1 row

struct Nms2dParams {
  const float* src;
  void* out;          // (planes, H, W): uint8 mask or fp32 values
  long long sB, sC;   // element strides of b and c in the source
  int C, H, W, tiles_x, tiles_y;
  long long tiles;    // planes * tiles_y * tiles_x
};

enum Nms3Mode { NMS3_MAX_MASK = 0, NMS3_MAX_VALUES = 1, NMS3_MINMAX = 2 };

struct Nms3dParams {
  const float* src;
  void* out0;             // (vols, L, H, W): the maxima (uint8 mask or fp32 values)
  void* out1;             // NMS3_MINMAX: the minima mask
  long long sB, sC, sL;   // element strides of b, c and the level in the source
  int C, L, H, W, tiles_x, tiles_y;
  long long tiles;        // vols * tiles_y * tiles_x
};

template <int K>
struct Nms2dShape {
  static constexpr int R = K / 2, SW = NMS_TW + 2 * R, SH = NMS_TH + 2 * R;
  // staged texels, K-column row maxima of every staged row, the same without the centre column on the tile's rows
  static constexpr int BYTES = (SH * SW + SH * NMS_TW + NMS_TH * NMS_TW) * 4;
};
constexpr int NMS3_SMEM_BYTES = (NMS3_TH + 2) * (NMS3_TW + 2) * 4;

__device__ __forceinline__ float nan_max(float a, float b) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#else
  return a != a ? a : b != b ? b : a > b ? a : b;
#endif
}

__device__ __forceinline__ float nan_min(float a, float b) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#else
  return a != a ? a : b != b ? b : a < b ? a : b;
#endif
}

// Four adjacent outputs of one row: uchar4 / float4 when the group lies in the row and is aligned, else one by one.
template <bool VALUES>
__device__ __forceinline__ void nms_store4(void* out, long long off, int gx, int W, const bool keep[4], const float c[4]) {
  if (VALUES) {
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = __fmul_rn(c[i], keep[i] ? 1.f : 0.f);
    float* o = static_cast<float*>(out) + off;
    if (gx + 3 < W && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (gx + i < W) o[i] = v[i];
    }
  } else {
    unsigned char* o = static_cast<unsigned char*>(out) + off;
    if (gx + 3 < W && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
      *reinterpret_cast<uchar4*>(o) = make_uchar4(keep[0], keep[1], keep[2], keep[3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (gx + i < W) o[i] = keep[i];
    }
  }
}

template <int K, bool VALUES>
__global__ void __launch_bounds__(NMS_NT) nms2d_kernel(const Nms2dParams p) {
  using S = Nms2dShape<K>;
  constexpr int R = S::R, SW = S::SW, SH = S::SH;
  constexpr bool GENERAL = K > 7;
  extern __shared__ __align__(128) unsigned char nms_smem[];
  float* s_src = reinterpret_cast<float*>(nms_smem);
  float* s_row = s_src + SH * SW;
  float* s_mid = s_row + SH * NMS_TW;
  const int tid = threadIdx.x;
  const int c4 = (tid & 15) * 4;
  for (long long t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    const int tx = (int)(t % p.tiles_x);
    const long long rest = t / p.tiles_x;
    const int ty = (int)(rest % p.tiles_y);
    const int plane = (int)(rest / p.tiles_y);
    const int x0 = tx * NMS_TW, y0 = ty * NMS_TH;
    const float* src = p.src + (long long)(plane / p.C) * p.sB + (long long)(plane % p.C) * p.sC;
    __syncthreads();  // the previous tile's readers are done with shared memory
    for (int i = tid; i < SH * SW; i += NMS_NT) {
      const int ly = i / SW, lx = i - ly * SW;
      const int gy = min(max(y0 - R + ly, 0), p.H - 1), gx = min(max(x0 - R + lx, 0), p.W - 1);
      float v = ldg(src + (long long)gy * p.W + gx);
      if (GENERAL && !(fabsf(v) <= 3.402823466e38f)) v = __int_as_float(0x7fffffff);  // not finite
      s_src[i] = v;
    }
    __syncthreads();
    for (int i = tid; i < SH * NMS_TW; i += NMS_NT) {
      const int ly = i / NMS_TW, lx = i - ly * NMS_TW;
      const float* row = s_src + ly * SW + lx;
      float left = row[0], right = row[R + 1];
#pragma unroll
      for (int j = 1; j < R; ++j) {
        left = nan_max(left, row[j]);
        right = nan_max(right, row[R + 1 + j]);
      }
      const float mid = nan_max(left, right);
      s_row[i] = nan_max(mid, row[R]);
      if (ly >= R && ly < R + NMS_TH) s_mid[i - R * NMS_TW] = mid;
    }
    __syncthreads();
    for (int ry = tid >> 4; ry < NMS_TH; ry += 16) {
      const int gy = y0 + ry, gx = x0 + c4;
      if (gy >= p.H || gx >= p.W) break;
      const float4 mm = *reinterpret_cast<const float4*>(s_mid + ry * NMS_TW + c4);
      float m[4] = {mm.x, mm.y, mm.z, mm.w};
#pragma unroll
      for (int dy = 0; dy < K; ++dy) {
        if (dy == R) continue;
        const float4 v = *reinterpret_cast<const float4*>(s_row + (ry + dy) * NMS_TW + c4);
        m[0] = nan_max(m[0], v.x);
        m[1] = nan_max(m[1], v.y);
        m[2] = nan_max(m[2], v.z);
        m[3] = nan_max(m[3], v.w);
      }
      const bool row_in = GENERAL || (gy >= R && gy < p.H - R);
      bool keep[4];
      float c[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        c[i] = s_src[(ry + R) * SW + c4 + i + R];
        if (GENERAL) keep[i] = c[i] > nan_max(m[i], 0.f);
        else keep[i] = row_in && gx + i >= R && gx + i < p.W - R && c[i] > m[i];
      }
      nms_store4<VALUES>(p.out, ((long long)plane * p.H + gy) * p.W + gx, gx, p.W, keep, c);
    }
  }
}

// One level of the 3-D walk: stage the 128 x 8 tile at (x0, y0) of the dense H x W plane `lev` plus a one-texel halo,
// replicate-clamped, in `s`; then reduce this thread's 4 columns (c4, row ry): the centre values, the 3 x 3 max and the
// 8-neighbour max (and with MIN the same minima).  Shared by nms3d_kernel and the sub-pixel refinement kernel
// (quad_interp.cuh), which computes its NMS mask on the same walk.
template <bool MIN>
__device__ __forceinline__ void nms3_stage_level(float* s, const float* lev, int H, int W, int x0, int y0, int tid, int c4, int ry,
                                                 float nval[4], float nmax[4], float n8max[4], float nmin[4], float n8min[4]) {
  constexpr int SW = NMS3_TW + 2, SH = NMS3_TH + 2;
  __syncthreads();  // the previous level's readers are done with shared memory
  for (int i = tid; i < SH * SW; i += NMS3_NT) {
    const int ly = i / SW, lx = i - ly * SW;
    const int yy = min(max(y0 - 1 + ly, 0), H - 1), xx = min(max(x0 - 1 + lx, 0), W - 1);
    s[i] = ldg(lev + (long long)yy * W + xx);
  }
  __syncthreads();
  float vmax[6], vmin[6], top[4], bot[4];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float a = s[ry * SW + c4 + j], b = s[(ry + 1) * SW + c4 + j], d = s[(ry + 2) * SW + c4 + j];
    vmax[j] = nan_max(nan_max(a, b), d);
    vmin[j] = nan_min(nan_min(a, b), d);
    if (j >= 1 && j <= 4) {
      top[j - 1] = a;
      bot[j - 1] = d;
      nval[j - 1] = b;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float side_max = nan_max(vmax[i], vmax[i + 2]), side_min = nan_min(vmin[i], vmin[i + 2]);
    nmax[i] = nan_max(side_max, vmax[i + 1]);
    n8max[i] = nan_max(side_max, nan_max(top[i], bot[i]));
    if (MIN) {
      nmin[i] = nan_min(side_min, vmin[i + 1]);
      n8min[i] = nan_min(side_min, nan_min(top[i], bot[i]));
    }
  }
}

// The 26-neighbour test of the ring's middle level: its centre against the 3 x 3 max of the levels either side and its
// own 8-neighbour max.
__device__ __forceinline__ bool nms3_is_max(float c, float below_max, float c8max, float above_max) {
  return c > nan_max(nan_max(below_max, c8max), above_max);
}

// 4 CTAs per SM: without the bound ptxas gives the minmax form 79 registers and 3 CTAs
template <int MODE>
__global__ void __launch_bounds__(NMS3_NT, 4) nms3d_kernel(const Nms3dParams p) {
  constexpr bool MINMAX = MODE == NMS3_MINMAX, VALUES = MODE == NMS3_MAX_VALUES;
  extern __shared__ __align__(128) unsigned char nms_smem[];
  float* s = reinterpret_cast<float*>(nms_smem);
  const int tid = threadIdx.x;
  const int c4 = (tid & 31) * 4, ry = tid >> 5;
  for (long long t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    const int tx = (int)(t % p.tiles_x);
    const long long rest = t / p.tiles_x;
    const int ty = (int)(rest % p.tiles_y);
    const int vol = (int)(rest / p.tiles_y);
    const int x0 = tx * NMS3_TW, y0 = ty * NMS3_TH;
    const int gy = y0 + ry, gx = x0 + c4;
    const bool active = gy < p.H && gx < p.W;
    const bool row_in = gy >= 1 && gy < p.H - 1;
    const float* src = p.src + (long long)(vol / p.C) * p.sB + (long long)(vol % p.C) * p.sC;
    // the ring: 3 x 3 max / min of level l - 2, and of level l - 1 its centre, 3 x 3 and 8-neighbour max / min
    float pmax[4] = {}, pmin[4] = {}, cmax[4] = {}, cmin[4] = {}, c8max[4] = {}, c8min[4] = {}, cval[4] = {};
    for (int l = 0; l <= p.L; ++l) {
      float nmax[4] = {}, nmin[4] = {}, n8max[4] = {}, n8min[4] = {}, nval[4] = {};
      if (l < p.L) nms3_stage_level<MINMAX>(s, src + (long long)l * p.sL, p.H, p.W, x0, y0, tid, c4, ry, nval, nmax, n8max, nmin, n8min);
      if (l >= 1 && active) {  // level l - 1 is complete: False on the border levels (l - 1 == 0 or l == L)
        const bool level_in = l >= 2 && l < p.L && row_in;
        bool kmax[4], kmin[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const bool in = level_in && gx + i >= 1 && gx + i < p.W - 1;
          kmax[i] = in && nms3_is_max(cval[i], pmax[i], c8max[i], nmax[i]);
          kmin[i] = in && cval[i] < nan_min(nan_min(pmin[i], c8min[i]), nmin[i]);
        }
        const long long off = (((long long)vol * p.L + (l - 1)) * p.H + gy) * p.W + gx;
        nms_store4<VALUES>(p.out0, off, gx, p.W, kmax, cval);
        if (MINMAX) nms_store4<false>(p.out1, off, gx, p.W, kmin, cval);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        pmax[i] = cmax[i];
        pmin[i] = cmin[i];
        cmax[i] = nmax[i];
        cmin[i] = nmin[i];
        c8max[i] = n8max[i];
        c8min[i] = n8min[i];
        cval[i] = nval[i];
      }
    }
  }
}

int nms2d_forward(const float* x, void* out, int B, int C, int H, int W, long long sB, long long sC, int k, bool values, cudaStream_t st);
int nms3d_forward(const float* x, void* out0, void* out1, int B, int C, int L, int H, int W, long long sB, long long sC, long long sL,
                  int mode, cudaStream_t st);

}  // namespace kb200
