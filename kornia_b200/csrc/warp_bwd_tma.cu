// kornia_b200 -- host dispatch of the tiled warp backward kernel.
#include "warp_bwd_tma.cuh"

namespace kb200 {

// KB200_EUNSUPPORTED -> the caller runs warp_bwd_generic.
int warp_tma_backward(const float* gout, const float* src, const float* m, const float* bx, const float* by, float* gsrc,
                             float* gm, void* workspace, int B, int C, int H, int W, int h, int w, int Bm, int projective, int interp,
                             int pad, int align, cudaStream_t st) {
  if (!option(OPT_TMA)) return KB200_EUNSUPPORTED;
  if (interp != KB200_BILINEAR || (pad != KB200_ZEROS && pad != KB200_BORDER) || (C != 3 && C != 1)) return KB200_EUNSUPPORTED;
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(src) & 15) != 0 || (gsrc && (reinterpret_cast<uintptr_t>(gsrc) & 15) != 0))
    return KB200_EUNSUPPORTED;
  if ((long long)B * C > 0x7fffffffll || (long long)B * ceil_div(h, 32) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  if ((w & 1) != 0 || (reinterpret_cast<uintptr_t>(gout) & 7) != 0) return KB200_EUNSUPPORTED;  // 8-byte loads of gout
  CUtensorMap mgsrc;  // unused when gsrc is null, but must encode
  if (!encode_plane_map(&mgsrc, gsrc ? gsrc : src, (long long)B * C, H, W, 72, BWD_SH, C)) return KB200_EUNSUPPORTED;
  CUtensorMap mgout;
  if ((w % 4) != 0 || (reinterpret_cast<uintptr_t>(gout) & 15) != 0 || !encode_plane_map(&mgout, gout, (long long)B * C, h, w, 64, 32, C))
    return KB200_EUNSUPPORTED;
  TmaBwdParams p{};
  p.gout = gout; p.src = src; p.m = m; p.bx = bx; p.by = by; p.gsrc = gsrc;
  p.B = B; p.H = H; p.W = W; p.h = h; p.w = w; p.Bm = Bm;
  p.max_segs = bwd_tma_max_segs(B, h);
  size_t rows = (size_t)bwd_tma_grid(B, h) * p.max_segs;
  // run-time work distribution (warp_bwd_tma2<DYN>): RGB, stride-1 lanes, enough strips to go round several times
  const bool dyn = C == 3 && option(OPT_DYN_SCHED) && option(OPT_BWD_STRIDE1) && (long long)B * ceil_div(h, 32) >= 4ll * bwd_tma_grid(B, h) &&
                   bwd_tma_dyn_chunks(B, h, w) * TMA_CONSUMER_WARPS < 0x7fffffffll;
  if (dyn) rows = (size_t)bwd_tma_dyn_chunks(B, h, w);  // one record row per chunk, all of them written
  if (gm) {
    p.records = reinterpret_cast<float*>(workspace);
    p.record_batch = reinterpret_cast<int*>(reinterpret_cast<char*>(workspace) + rows * TMA_CONSUMER_WARPS * 9 * sizeof(float));
  }
  CUtensorMap msrcwin;
  if (!encode_plane_map(&msrcwin, src, (long long)B * C, H, W, 72, BWD_SH, C)) return KB200_EUNSUPPORTED;
  if (dyn) {
    p.counter = take_work_counter(st);
    if (!p.counter) return KB200_EUNSUPPORTED;
    p.chunk_tiles = BWD_DYN_CHUNK;
  }
  const int rc = launch_warp_bwd_tma2(msrcwin, mgsrc, mgout, p, C, pad, projective, align, gsrc != nullptr, gm != nullptr, dyn, st);
  if (rc != KB200_OK || !gm) return rc;
  warp_gm_reduce_records<<<dim3(9, Bm), 256, 0, st>>>(p.records, p.record_batch, gm, (int)rows, Bm,
                                                        dyn ? (int)(rows / (size_t)B) : 0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("warp_gm_reduce_records launch failed: %s", cudaGetErrorString(e));
    return KB200_ECUDA;
  }
  return KB200_OK;
}

}  // namespace kb200
