// kornia_b200 -- one octave of ScalePyramid in one pass: every blur level of an octave, walking DOWN column bands (fp32).
//
// Replaces the per-level loop of kornia/geometry/transform/pyramid.py:367-384 (ScalePyramid._blur_fast: F.pad + F.conv2d
// twice per level, then torch.stack).  Level 0 is the source (copy stage) or its reflect-bordered separable blur with the
// initial taps (blur stage); level l >= 1 is the reflect-bordered separable blur of level l - 1.  The kernel reads the
// source once and writes the (planes, L, H, W) stack; no level goes back to HBM.
//
// Persistent CTAs walk 128-column bands top to bottom in steps of TH = 16 rows.  The blur chain is a pipeline of stages:
// at step t stage l takes the TH rows of level l - 1 that stage l - 1 just produced, row-filters them into its ring of
// TH + K_l - 1 row-filtered rows (a circular buffer: the K_l - 1 rows shared with the next step stay where they are), and
// column-filters the ring into TH rows of level l, D_l = r_0 + ... + r_l rows above the source rows of that step.  So no
// row is filtered twice vertically.  Horizontally, level l is computed on the band plus E_l = r_{l+1} + ... + r_{L-1}
// columns on each side (the support of the levels after it); only the band's columns are stored.
//
// Arithmetic is the composition's (filter2d_separable per level, sepfilter_tiled_kernel / sepfilter_fwd_generic): a row
// pass, then a column pass, each with ascending taps, __fmaf_rn, from 0.  The reflect border belongs to each level's
// computed values: out-of-image columns of a level and out-of-image row-filtered rows are copies of their reflections
// (a row filter works row by row, so a reflected row-filtered row equals the row filter of the reflected row).  The
// source is loaded with the reflection already applied.  Only the columns and rows within the next stage's radius of
// the image are patched: cells farther out feed only cells that are out of the image themselves, which are patched or
// never read.  Bit-identical to the per-level composition, -0 and NaN included.
//
// A segment of a band that starts at step t0 > 0 (more CTAs than bands) first runs PRIME steps without storing, so
// every ring holds what a walk from the top would hold.
//
// Launched by octave_vwalk.cu; tests/test_scale_pyramid_gpu.py checks it bit for bit against the composition, and
// tools/hostemu (run_emu --octave) runs it on the host.
#pragma once
#include "filter_generic.cuh"
#include "tma.cuh"

namespace kb200 {

constexpr int OCT_BW = 128;     // band width (stored columns per CTA)
constexpr int OCT_TH = 16;      // rows per step
constexpr int OCT_NT = 512;     // threads per CTA
constexpr int OCT_MAX_L = 6;    // levels per octave
constexpr int OCT_MAX_K = 25;   // taps per level

struct OctaveParams {
  const float* src;  // (planes,H,W)
  float* out;        // (planes,L,H,W)
  int planes, H, W;
  float taps[OCT_MAX_L][OCT_MAX_K];  // [stage][tap]: stage 0 the initial blur (blur stage only), stage l the level l-1 -> l taps
};

__host__ __device__ constexpr int oct_round4(int v) { return (v + 3) & ~3; }

// Compile-time layout of a chain.  K0 = 0: copy stage (level 0 is the source); else the initial blur's tap count.
template <int K0, int... KS>
struct OctaveChain {
  static constexpr int L = 1 + sizeof...(KS);
  static constexpr bool BLUR0 = K0 > 0;
  static constexpr int K[L] = {K0 > 0 ? K0 : 1, KS...};
  static_assert(L <= OCT_MAX_L, "levels");
  __host__ __device__ static constexpr int r(int l) { return (K[l] - 1) / 2; }
  // columns computed on each side of the band at level l (l = -1: the source)
  __host__ __device__ static constexpr int E(int l) {
    int e = 0;
    for (int m = l + 1; m < L; ++m) e += r(m);
    return e;
  }
  // rows level l lags the source rows of a step
  __host__ __device__ static constexpr int D(int l) {
    int d = 0;
    for (int m = 0; m <= l; ++m) d += r(m);
    return d;
  }
  __host__ __device__ static constexpr int WID(int l) { return OCT_BW + 2 * E(l); }      // computed columns of level l
  __host__ __device__ static constexpr int STRIDE(int l) { return oct_round4(WID(l) + 3); }  // the 4-wide row pass reads up to 3 past the end
  __host__ __device__ static constexpr int RING(int l) { return OCT_TH + K[l] - 1; }
  __host__ __device__ static constexpr bool HAS_RING(int l) { return l > 0 || BLUR0; }
  // steps before a segment's first stored step that refill every ring
  __host__ __device__ static constexpr int PRIME() {
    int p = 0;
    for (int l = 0; l < L; ++l)
      if (HAS_RING(l)) p += (K[l] - 1 + OCT_TH - 1) / OCT_TH;
    return p;
  }
  // shared memory, in floats: source rows, two level buffers, the rings
  static constexpr int SRC_OFF = 0;
  __host__ __device__ static constexpr int LEV_STRIDE() {
    int s = 0;
    for (int l = 0; l < L; ++l) s = s > STRIDE(l) ? s : STRIDE(l);
    return s;
  }
  static constexpr int LEV_OFF = SRC_OFF + OCT_TH * STRIDE(-1);
  __host__ __device__ static constexpr int RING_OFF(int l) {
    int o = LEV_OFF + 2 * OCT_TH * LEV_STRIDE();
    for (int m = 0; m < l; ++m)
      if (HAS_RING(m)) o += RING(m) * STRIDE(m);
    return o;
  }
  __host__ __device__ static constexpr int FLOATS() { return RING_OFF(L); }
  __host__ __device__ static constexpr size_t SMEM_BYTES() { return (size_t)FLOATS() * sizeof(float); }
  static constexpr int SRC_PER_THREAD = (OCT_TH * STRIDE(-1) + OCT_NT - 1) / OCT_NT;
};

// reflect index of q on [0, n), for the q the walk reads; q far outside (cells nobody uses) is clamped first
__device__ __forceinline__ int oct_fold(int q, int n) {
  q = q < -(n - 1) ? -(n - 1) : (q > 2 * (n - 1) ? 2 * (n - 1) : q);
  return border_index<KB200_REFLECT>(q, n);
}

// row pass of stage l: TH rows of `in` (level l - 1, columns from E(l-1) left of the band) -> ring rows at pos0 ...
template <typename CH, int l>
__device__ __forceinline__ void oct_row_pass(const OctaveParams& p, const float* in, float* ring, int pos0) {
  constexpr int K = CH::K[l], IS = CH::STRIDE(l - 1), OS = CH::STRIDE(l), R = CH::RING(l);
  constexpr int Q = (CH::WID(l) + 3) / 4;
  for (int e = threadIdx.x; e < OCT_TH * Q; e += OCT_NT) {
    const int o = e / Q, q = e - o * Q;
    const float* src = in + o * IS + 4 * q;
    float win[K + 3];
#pragma unroll
    for (int j = 0; j < K + 3; ++j) win[j] = src[j];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < K; ++j)
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] = __fmaf_rn(p.taps[l][j], win[j + u], acc[u]);
    int pos = pos0 + o;
    if (pos >= R) pos -= R;
    *reinterpret_cast<float4*>(ring + pos * OS + 4 * q) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
}

// input of stage l: the source rows (stage 0; stage 1 of a copy chain, whose level 0 is the source), else level l - 1
template <typename CH, int l>
__device__ __forceinline__ const float* oct_input(float* smem) {
  constexpr int LEV = CH::LEV_OFF + ((l - 1) & 1) * OCT_TH * CH::LEV_STRIDE();
  if constexpr (l == 0 || (l == 1 && !CH::BLUR0)) return smem + CH::SRC_OFF;
  else return smem + LEV;
}

// stage l of step t (rows of level l: t*TH - D(l) ...), then stages l+1 ...
template <typename CH, int l>
__device__ __forceinline__ void oct_stage(const OctaveParams& p, float* smem, size_t plane, int x0, int t, bool store) {
  if constexpr (l < CH::L) {
    constexpr int OS = CH::STRIDE(l), R = CH::RING(l), C = CH::K[l] - 1, K = CH::K[l];
    constexpr int E = CH::E(l), WID = CH::WID(l), DL = CH::D(l), LS = CH::LEV_STRIDE(), LEV_OFF = CH::LEV_OFF;
    constexpr int SS = CH::STRIDE(-1), RING_OFF = CH::RING_OFF(l), NL = CH::L;
    const int H = p.H, W = p.W;
    const int y0 = t * OCT_TH - DL;  // image row of this step's first row of level l
    float* lev = smem + LEV_OFF + (l & 1) * OCT_TH * LS;
    if constexpr (!CH::HAS_RING(l)) {
      // copy stage: level 0 is the source as loaded (rows t*TH ..., columns E(-1) = E(0) left of the band)
      if (store) {
        for (int e = threadIdx.x; e < OCT_TH * (OCT_BW / 4); e += OCT_NT) {
          const int o = e / (OCT_BW / 4), c = 4 * (e - o * (OCT_BW / 4));
          const int gy = y0 + o, gx = x0 + c;
          const float* s = smem + CH::SRC_OFF + o * SS + E + c;
          if (gy >= 0 && gy < H && gx < W)
            __stcs(reinterpret_cast<float4*>(p.out + ((plane * NL + l) * H + gy) * (size_t)W + gx), make_float4(s[0], s[1], s[2], s[3]));
        }
      }
    } else {
      float* ring = smem + RING_OFF;
      const int base = (t * OCT_TH) % R;  // ring position of ring row 0 (image row y0 - r)
      int pos0 = base + C;
      if (pos0 >= R) pos0 -= R;
      oct_row_pass<CH, l>(p, oct_input<CH, l>(smem), ring, pos0);
      __syncthreads();
      // reflect border of the row-filtered rows: ring row i is image row g = y0 - r + i
      const int g0 = y0 - C / 2;
      if (g0 < 0 || g0 + R > H) {  // CTA-uniform
        constexpr int Q = OS / 4;
        for (int e = threadIdx.x; e < R * Q; e += OCT_NT) {
          const int i = e / Q, q = e - i * Q;
          const int g = g0 + i;
          if (g >= 0 && g < H) continue;
          if (g < -(C / 2) || g >= H + C / 2) continue;  // beyond the radius: never read for an in-image row
          const int si = border_index<KB200_REFLECT>(g, H) - g0;
          if ((unsigned)si >= (unsigned)R) continue;
          int pd = base + i, ps = base + si;
          if (pd >= R) pd -= R;
          if (ps >= R) ps -= R;
          reinterpret_cast<float4*>(ring + pd * OS)[q] = reinterpret_cast<const float4*>(ring + ps * OS)[q];
        }
        __syncthreads();
      }
      // column pass: 4 rows x 1 column per item
      constexpr int RY = 4;
      for (int e = threadIdx.x; e < (OCT_TH / RY) * WID; e += OCT_NT) {
        const int rg = e / WID, c = e - rg * WID;
        float acc[RY];
#pragma unroll
        for (int u = 0; u < RY; ++u) acc[u] = 0.f;
#pragma unroll
        for (int i = 0; i < RY + K - 1; ++i) {
          int pos = base + rg * RY + i;
          if (pos >= R) pos -= R;
          const float v = ring[pos * OS + c];
#pragma unroll
          for (int u = 0; u < RY; ++u)
            if (i - u >= 0 && i - u < K) acc[u] = __fmaf_rn(p.taps[l][i - u], v, acc[u]);
        }
        const int gx = x0 - E + c;
#pragma unroll
        for (int u = 0; u < RY; ++u) {
          const int o = rg * RY + u;
          lev[o * OS + c] = acc[u];
          const int gy = y0 + o;
          if (store && c >= E && c < E + OCT_BW && gx < W && gy >= 0 && gy < H)
            __stcs(p.out + ((plane * NL + l) * H + gy) * (size_t)W + gx, acc[u]);
        }
      }
      __syncthreads();
      // reflect border of level l's columns, within the next stage's radius
      if constexpr (l + 1 < CH::L) {
        constexpr int RN = CH::r(l + 1);
        if (x0 - E < 0 || x0 - E + WID > W) {  // CTA-uniform
          for (int e = threadIdx.x; e < OCT_TH * 2 * RN; e += OCT_NT) {
            const int o = e / (2 * RN), k = e - o * (2 * RN);
            const int g = k < RN ? -1 - k : W + (k - RN);  // columns -1 .. -RN, W .. W + RN - 1
            const int c = g - (x0 - E), sc = border_index<KB200_REFLECT>(g, W) - (x0 - E);
            if ((unsigned)c < (unsigned)WID && (unsigned)sc < (unsigned)WID) lev[o * OS + c] = lev[o * OS + sc];
          }
          __syncthreads();
        }
      }
    }
    oct_stage<CH, l + 1>(p, smem, plane, x0, t, store);
  }
}

template <typename CH>
__global__ void __launch_bounds__(OCT_NT, 1) octave_vwalk_kernel(const __grid_constant__ OctaveParams p) {
  extern __shared__ __align__(128) unsigned char oct_smem[];
  float* smem = reinterpret_cast<float*>(oct_smem);
  constexpr int SS = CH::STRIDE(-1), ES = CH::E(-1), NPT = CH::SRC_PER_THREAD, DEPTH = CH::D(CH::L - 1), PRIME = CH::PRIME();
  const int H = p.H, W = p.W;
  const int bands = ceil_div(W, OCT_BW), steps = ceil_div(H + DEPTH, OCT_TH);
  const Segments segs(p.planes * bands, steps);

  // source rows of step t, reflected, into registers (issued a step ahead of their use)
  float pre[NPT];
  auto fetch = [&](int strip, int t) {
    const int plane = strip / bands, x0 = (strip - plane * bands) * OCT_BW;
    const float* src = p.src + (size_t)plane * H * W;
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
      const int e = threadIdx.x + k * OCT_NT;
      const int o = e / SS, c = e - o * SS;
      if (o < OCT_TH) pre[k] = __ldg(src + (size_t)oct_fold(t * OCT_TH + o, H) * W + oct_fold(x0 - ES + c, W));
    }
  };
  auto put = [&]() {
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
      const int e = threadIdx.x + k * OCT_NT;
      if (e < OCT_TH * SS) smem[CH::SRC_OFF + e] = pre[k];
    }
  };

  int strip, t0, t1, cursor = 0;
  for (int seg = 0; segs.get(seg, strip, t0, t1, cursor); ++seg) {
    const int plane = strip / bands, x0 = (strip - plane * bands) * OCT_BW;
    const int s0 = t0 - PRIME > 0 ? t0 - PRIME : 0;
    fetch(strip, s0);
    __syncthreads();  // the previous segment's last step is done with the source rows
    put();
    __syncthreads();
    for (int t = s0; t < t1; ++t) {
      if (t + 1 < t1) fetch(strip, t + 1);
      oct_stage<CH, 0>(p, smem, (size_t)plane, x0, t, t >= t0);
      if (t + 1 < t1) {
        put();  // every stage has synchronised after its last read of the source rows
        __syncthreads();
      }
    }
  }
}

// host entry (octave_vwalk.cu).  ksizes[0] is the initial blur's tap count (0: level 0 is the source), ksizes[1 .. L-1]
// the level kernels; taps holds them in that order.  KB200_EUNSUPPORTED outside the envelope (a chain that is not
// instantiated, a tap count above min(H, W), rows that are not a multiple of 4 floats, misaligned buffers).
int octave_vwalk_forward(const float* x, const double* taps, const int* ksizes, int L, float* out, int planes, int H, int W, cudaStream_t st);

}  // namespace kb200
