// kornia_b200 -- host-side launch helpers of the TMA-tiled warp forward kernel (included by the
// per-interpolation translation units warp_tma_{bilinear,nearest,bicubic}.cu so they compile in parallel).
#pragma once
#include "warp_tma.cuh"

namespace kb200 {

constexpr int TMA_L2_PROMO = 256;  // 256-B L2 promotion on the tensor map (not compared with 128 B on the H100)

// 64 x 32 output tiles, 72-wide source boxes of 33 to 40 rows, 2 stages, 2 CTAs per SM: not compared with 3 stages, 96-wide
// boxes or other tiles on the H100.  On an H100 SXM (700 W) the headline launch ran at 0.77 of the 3.35 TB/s roofline under
// the strip deal (4.95 ms; 5.36 ms with the 40-row box for every tile).  DYN launches run the sweep by default (every tile
// drawn in raster order): on an H100 held to 400 W, 4.47-4.55 ms against 4.95-4.97 ms for the strip deal.  Column-wise walks
// of bands of strips were measured and lost (DESIGN.md 4.1).
template <int NC, int INTERP, int PAD, bool PROJ, bool ALIGN, int TW = 64, int TH = 32, int BW = 72, int BH = 40, int NSTAGE = 2, bool DYN = false>
static int launch_warp_tma(const TmaBoxMaps& maps, const TmaWarpParams& p, cudaStream_t st, int ctas_per_sm = 2) {
  auto kern = warp_fwd_tma<NC, INTERP, PAD, PROJ, ALIGN, TW, TH, BW, BH, NSTAGE, DYN>;
  constexpr size_t smem = NSTAGE * (size_t)NC * BW * BH * 4 + 2 * NSTAGE * sizeof(uint64_t) + NSTAGE * sizeof(StageInfo) + NSTAGE * 12 * sizeof(float);
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, smem);
  const long long nstrips = (long long)p.B * ceil_div(p.h, TH);
  const long long cap = (long long)ctas_per_sm * sm_count();
  const int grid = (int)(nstrips < cap ? nstrips : cap);
  if (DYN) {
    TmaWarpParams q = p;
    q.counter = take_work_counter(st);
    if (!q.counter) return KB200_EUNSUPPORTED;
    if (option(OPT_SWEEP)) {  // every run drawn, in raster order (warp_fwd_tma: the producer)
      q.chunk_tiles = SWEEP_TILES;
      q.static_pct = 0;
    } else {
      q.chunk_tiles = option(OPT_DYN_CHUNK) > 0 ? option(OPT_DYN_CHUNK) : 10;
      q.static_pct = option(OPT_DYN_STATIC);
    }
    kern<<<grid, TMA_THREADS, smem, st>>>(maps, q);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("warp_fwd_tma<DYN> launch failed: %s", cudaGetErrorString(e));
      return KB200_ECUDA;
    }
    return KB200_OK;
  }
  kern<<<grid, TMA_THREADS, smem, st>>>(maps, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("warp_fwd_tma launch failed: %s", cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

// Returns KB200_EUNSUPPORTED when the request is outside this kernel's envelope (the caller then
// uses warp_fwd_generic): non-bilinear, fill padding, C > 4, rows not 16-byte aligned.

struct TmaFwdArgs {
  const float *src, *m, *bx, *by, *fill;
  float* out;
  int B, C, H, W, h, w, Bm, projective, pad, align;
  int only_class;  // 0: all samples; CLASS_WIDE / CLASS_SQUARE: only the samples of that footprint class
};

// The source as (W, H, B * C) planes, one map per box height of warp_fwd_tma (tma_box_rows); false when the driver refuses.
template <int BW, int BH>
static bool encode_box_maps(TmaBoxMaps& maps, const TmaFwdArgs& a) {
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.B * a.C};
  const cuuint64_t strides[2] = {(cuuint64_t)a.W * 4, (cuuint64_t)a.H * a.W * 4};
  const cuuint32_t estr[3] = {1, 1, 1};
  for (int i = 0; i < TMA_BOX_HEIGHTS; ++i) {
    const cuuint32_t box[3] = {(cuuint32_t)BW, (cuuint32_t)tma_box_rows(BH, i), 1};
    if (encode(&maps.map[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(a.src), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
  }
  return true;
}

template <int INTERP>
static int warp_tma_forward_impl(const TmaFwdArgs& a, cudaStream_t st) {
  TmaBoxMaps map;
  if (!encode_box_maps<72, 40>(map, a)) return KB200_EUNSUPPORTED;
  TmaWarpParams p{a.src, a.m, a.bx, a.by, a.fill, a.out, a.B, a.H, a.W, a.h, a.w, a.Bm, a.align, a.only_class, nullptr, 0, 0};
  const int C = a.C, pad = a.pad;
  const bool projective = a.projective != 0, align = a.align != 0;
  // run-time work distribution (warp_fwd_tma<DYN>) for bilinear RGB batches with enough strips to go round several times
  if constexpr (INTERP == KB200_BILINEAR)
    if (C == 3 && option(OPT_DYN_SCHED) && (long long)a.B * ceil_div(a.h, 32) >= 8ll * sm_count() && ceil_div(a.w, 64) < 32768 &&
        (long long)a.B * ceil_div(a.h, 32) * ceil_div(a.w, 64) < 0x7fffffffll) {
      int rc = KB200_EUNSUPPORTED;
#define KB_TMA_DYN_CASE(PAD_)                                                                                                     \
  if (pad == PAD_)                                                                                                                \
    rc = projective ? (align ? launch_warp_tma<3, INTERP, PAD_, true, true, 64, 32, 72, 40, 2, true>(map, p, st)                \
                             : launch_warp_tma<3, INTERP, PAD_, true, false, 64, 32, 72, 40, 2, true>(map, p, st))              \
                    : (align ? launch_warp_tma<3, INTERP, PAD_, false, true, 64, 32, 72, 40, 2, true>(map, p, st)               \
                             : launch_warp_tma<3, INTERP, PAD_, false, false, 64, 32, 72, 40, 2, true>(map, p, st));
      KB_TMA_DYN_CASE(KB200_ZEROS)
      KB_TMA_DYN_CASE(KB200_BORDER)
      KB_TMA_DYN_CASE(KB200_REFLECTION)
      KB_TMA_DYN_CASE(KB200_FILL)
#undef KB_TMA_DYN_CASE
      if (rc != KB200_EUNSUPPORTED) return rc;
    }
#define KB_TMA_CASE(NC_, PAD_)                                                                                                   \
  if (C == NC_ && pad == PAD_)                                                                                                   \
    return projective ? (align ? launch_warp_tma<NC_, INTERP, PAD_, true, true>(map, p, st)                                  \
                               : launch_warp_tma<NC_, INTERP, PAD_, true, false>(map, p, st))                                \
                      : (align ? launch_warp_tma<NC_, INTERP, PAD_, false, true>(map, p, st)                                 \
                               : launch_warp_tma<NC_, INTERP, PAD_, false, false>(map, p, st));
  KB_TMA_CASE(3, KB200_ZEROS)
  KB_TMA_CASE(3, KB200_BORDER)
  KB_TMA_CASE(3, KB200_REFLECTION)
  KB_TMA_CASE(3, KB200_FILL)
  KB_TMA_CASE(1, KB200_ZEROS)
  KB_TMA_CASE(1, KB200_BORDER)
  KB_TMA_CASE(1, KB200_REFLECTION)
  KB_TMA_CASE(1, KB200_FILL)
  if (INTERP == KB200_BILINEAR) {
    KB_TMA_CASE(4, KB200_ZEROS)
    KB_TMA_CASE(4, KB200_BORDER)
    KB_TMA_CASE(4, KB200_REFLECTION)
    KB_TMA_CASE(2, KB200_ZEROS)
    KB_TMA_CASE(2, KB200_BORDER)
    KB_TMA_CASE(2, KB200_REFLECTION)
  }
#undef KB_TMA_CASE
  return KB200_EUNSUPPORTED;
}

int warp_tma_forward_bilinear(const TmaFwdArgs& a, cudaStream_t st);
int warp_tma_forward_nearest(const TmaFwdArgs& a, cudaStream_t st);
int warp_tma_forward_bicubic(const TmaFwdArgs& a, cudaStream_t st);
// bilinear, C in {1,3}: 32 x 32 output tiles with a 56 x 56 source box, for the samples of class CLASS_SQUARE
int warp_tma_forward_square(const TmaFwdArgs& a, cudaStream_t st);

}  // namespace kb200
