// kornia_b200 -- shared pieces of the tiled fused warp backward kernels (fp32, bilinear, zeros/border, C = 3 or 1):
// parameters, the exact per-pixel path, the fixed-order second stage of d/dM and the host-side sizing.  The kernels are
// warp_bwd_tma2.cuh (every warp its own pipeline).
//
// Replaces grid_sampler_2d_backward (atomic scatter into a zero-filled tensor + a dense grad_grid) and the autograd of the
// ~15 broadcast elementwise ops of kornia/geometry/transform/imgwarp.py:165-170 (SURVEY.md appendix A.5).
//   * d/dsrc: every warp owns a private 72x8xC accumulation strip in shared memory; taps are added with plain LDS/FADD/STS
//     and the strip is added to global memory by ONE cp.reduce.async.bulk.tensor (TMA reduce-add, SASS UTMAREDG.3D.ADD) per
//     warp and tile instead of twelve scattered atomics per pixel; out-of-image cells are clipped by the TMA unit.
//     (A TMA reduce with a negative box coordinate traps, so strip origins are clamped to >= 0.)
//   * d/dM: taps come from a TMA-staged source window; the nine per-pixel partials accumulate in registers over a whole
//     strip segment, then warp-shuffle -> one record per (CTA, segment, warp); a second kernel sums the records in a fixed
//     order (deterministic, double accumulation).
#pragma once
#include "warp_tma.cuh"

namespace kb200 {

struct TmaBwdParams {
  const float* gout;   // (B,NC,h,w)
  const float* src;    // (B,NC,H,W)
  const float* m;      // (Bm,3,3)
  const float* bx;
  const float* by;
  float* gsrc;         // (B,NC,H,W) zero-filled by the caller, or null
  float* records;      // (grid, max_segs, 8 warps, 9) partial sums for d/dm, or null
  int* record_batch;   // (grid, max_segs) batch index of each record row, -1 = unused
  int B, H, W, h, w, Bm, max_segs;
  int* counter;        // DYN kernels only: zero-initialised work counter of this launch
  int chunk_tiles;     // DYN kernels only: tiles per chunk
};

constexpr int BWD_SH = 8;         // rows of a warp's accumulation strip
constexpr int BWD_THREADS = 256;  // 8 warps; warp 0 doubles as the TMA issuer (a 9th warp would cap registers at 96)

#ifdef KB200_HOST_EMU
static long long emu_exact_path_pixels = 0;
#endif

// One pixel handled entirely through global memory: exact scatter with bounds tests and, when
// requested, the coordinate gradient from global taps.  Returns (gix, giy).
template <int NC, int PAD, bool NEED_SRC, bool NEED_M>
__device__ __noinline__ float2 bwd_pixel_global(const TmaBwdParams& p, int b, int y, int x, float ix, float iy) {
#ifdef KB200_HOST_EMU
  ++emu_exact_path_pixels;  // tools/hostemu reports how many pixels left the shared-memory fast path
#endif
  const int H = p.H, W = p.W;
  const size_t splane = (size_t)H * W, oplane = (size_t)p.h * p.w;
  const float* gop = p.gout + (size_t)b * NC * oplane + (size_t)y * p.w + x;
  ix = guard_index(ix);  // NaN / inf / beyond int range -> out of bounds, as in the generic kernel
  iy = guard_index(iy);
  const float x0f = floorf(ix), y0f = floorf(iy);
  const float wx1 = (x0f + 1.f) - ix, wx0 = ix - x0f, wy1 = (y0f + 1.f) - iy, wy0 = iy - y0f;
  const int x0 = (int)x0f, y0 = (int)y0f;
  const bool ok_nw = in_bounds(y0, x0, H, W), ok_ne = in_bounds(y0, x0 + 1, H, W);
  const bool ok_sw = in_bounds(y0 + 1, x0, H, W), ok_se = in_bounds(y0 + 1, x0 + 1, H, W);
  const int o = y0 * W + x0;
  float gix = 0.f, giy = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const float go = __ldg(gop + c * oplane);
    if (NEED_SRC) {
      float* gs = p.gsrc + ((size_t)b * NC + c) * splane;
      if (ok_nw) atomicAdd(gs + o, wx1 * wy1 * go);
      if (ok_ne) atomicAdd(gs + o + 1, wx0 * wy1 * go);
      if (ok_sw) atomicAdd(gs + o + W, wx1 * wy0 * go);
      if (ok_se) atomicAdd(gs + o + W + 1, wx0 * wy0 * go);
    }
    if (NEED_M) {
      const float* s = p.src + ((size_t)b * NC + c) * splane;
      const float v_nw = ok_nw ? __ldg(s + o) : 0.f, v_ne = ok_ne ? __ldg(s + o + 1) : 0.f;
      const float v_sw = ok_sw ? __ldg(s + o + W) : 0.f, v_se = ok_se ? __ldg(s + o + W + 1) : 0.f;
      gix += go * ((v_ne - v_nw) * wy1 + (v_se - v_sw) * wy0);
      giy += go * ((v_sw - v_nw) * wx1 + (v_se - v_ne) * wx0);
    }
  }
  return make_float2(gix, giy);
}

// Second stage of d/dm for the tiled kernel: fixed-order sum over the record rows of each sample.
// grid = (9, Bm).  records (rows, 8, 9), record_batch (rows).
// rows_per_batch > 0 (the run-time work distribution: row = chunk, the chunks of a sample are consecutive): only that sample's rows.
static __global__ void __launch_bounds__(256) warp_gm_reduce_records(const float* __restrict__ records, const int* __restrict__ record_batch,
                                                              float* __restrict__ gm, int rows, int Bm, int rows_per_batch) {
  const int k = blockIdx.x, bm = blockIdx.y;
  double s = 0.0;
  const int r0 = (rows_per_batch > 0 && Bm != 1) ? bm * rows_per_batch : 0;
  const int r1 = (rows_per_batch > 0 && Bm != 1) ? r0 + rows_per_batch : rows;
  for (int r = r0 + threadIdx.x; r < r1; r += 256) {
    const int rb = record_batch[r];
    if (rb < 0 || (Bm != 1 && rb != bm)) continue;
    const float* rec = records + (size_t)r * TMA_CONSUMER_WARPS * 9 + k;
#pragma unroll
    for (int w = 0; w < TMA_CONSUMER_WARPS; ++w) s += (double)rec[w * 9];
  }
  __shared__ double sh[256];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) gm[(size_t)bm * 9 + k] = (float)sh[0];
}

// ------------------------------------------------------------------------------------------ host
inline int bwd_tma_grid(int B, int h) {
  const long long nstrips = (long long)B * ceil_div(h, 32);
  const long long cap = 2ll * sm_count();
  return (int)(nstrips < cap ? nstrips : cap);
}
inline int bwd_tma_max_segs(int B, int h) {
  const long long nstrips = (long long)B * ceil_div(h, 32);
  return (int)(nstrips / bwd_tma_grid(B, h)) + 2;
}
constexpr int BWD_DYN_CHUNK = 10;  // tiles per chunk of the run-time work distribution (warp_bwd_tma2<DYN>)
inline long long bwd_tma_dyn_chunks(int B, int h, int w) { return (long long)B * ceil_div(h, 32) * ceil_div(ceil_div(w, 64), BWD_DYN_CHUNK); }
inline size_t bwd_tma_workspace_bytes(int B, int h, int w) {  // record rows: one per (CTA, segment) of the static deal or one per chunk
  size_t rows = (size_t)bwd_tma_grid(B, h) * bwd_tma_max_segs(B, h);
  if ((size_t)bwd_tma_dyn_chunks(B, h, w) > rows) rows = (size_t)bwd_tma_dyn_chunks(B, h, w);
  return rows * (TMA_CONSUMER_WARPS * 9 * sizeof(float)) + rows * sizeof(int) + 256;
}

// msrcwin: tensor map of `src` with the per-warp window box (72, BWD_SH, C).
int launch_warp_bwd_tma2(const CUtensorMap& msrcwin, const CUtensorMap& mgsrc, const CUtensorMap& mgout, const TmaBwdParams& p, int C, int pad,
                         int projective, int align, bool need_src, bool need_m, bool dyn, cudaStream_t st);

int warp_tma_backward(const float* gout, const float* src, const float* m, const float* bx, const float* by, float* gsrc, float* gm,
                      void* workspace, int B, int C, int H, int W, int h, int w, int Bm, int projective, int interp, int pad, int align,
                      cudaStream_t st);

}  // namespace kb200
