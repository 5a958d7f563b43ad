// kornia_b200 -- the double-buffered TMA tile feed of the persistent tiled kernels (sepfilter_tiled, filter2d_tiled,
// filter2d_taps, gradient_tiled, ssim_vwalk, corner_vwalk).
//
// A CTA walks the tiles of its Segments in order; box n of that walk lands in slot n & 1 and completes on full[n & 1].
// Thread 0 issues the loads two boxes ahead of the consumers: two at the start, then one each time the CTA has finished
// with a slot.  The consumers count the boxes they take in their own n and wait with mbar_wait(&full[n & 1], (n >> 1) & 1).
// Band walkers (PROLOGUE) take one extra box before the first tile of each segment, at step t0 - 1, holding the rows
// that the segment's first tile carries in from above.
#pragma once
#include "filter_generic.cuh"
#include "tma.cuh"

namespace kb200 {

// Two slot barriers, one arrival (thread 0's expect_tx) per phase; every thread of the CTA returns after they are set up.
__device__ __forceinline__ void feed_init(uint64_t* full) {
  if (threadIdx.x == 0) {
    tma::mbar_init(&full[0], 1);
    tma::mbar_init(&full[1], 1);
    tma::fence_barrier_init();
  }
  __syncthreads();
}

// The issuing thread's copy of the CTA's walk.  load(slot, strip, t, prologue) is the kernel's own: it arms full[slot]
// with the box's bytes and issues the box of step t of `strip` (t is the tile index along the strip, t0 - 1 for a
// prologue box) into that slot.
template <bool PROLOGUE>
struct TileFeed {
  const Segments& segs;
  int seg = 0, strip = 0, t0 = 0, t1 = 0, cursor = 0, t = 0, n = 0;
  bool live = false;

  __device__ explicit TileFeed(const Segments& s) : segs(s) {}

  template <typename Load>
  __device__ void start(Load&& load) {
    next();  // -> the first box
    issue(load);
    issue(load);
  }
  // load the box the walk points at, then step
  template <typename Load>
  __device__ void issue(Load&& load) {
    if (!live) return;
    tma::fence_proxy_async();
    load(n & 1, strip, t, PROLOGUE && t < t0);
    next();
  }

 private:
  __device__ void next() {
    if (live && t + 1 < t1) {
      ++t;
      ++n;
      return;
    }
    // n counts boxes: the first box of the walk is box 0, so only later segment starts step it
    const bool first = !live && n == 0 && seg == 0;
    live = segs.get(seg, strip, t0, t1, cursor);
    ++seg;
    t = PROLOGUE ? t0 - 1 : t0;
    if (!first) ++n;
  }
};

// 'reflect' / 'replicate' on a box that sticks out of the image (CTA-uniform test): each out-of-image cell of the
// (rows x bw) box at image position (ox, oy) of the p.H x p.W image (p: the kernel's parameters) copies the cell it folds
// to, where that lies in the box, then the CTA synchronises.  Cells whose fold lies outside the box are left alone; the
// callers never read them.  'constant' needs no patch: TMA fills out-of-image texels with zeros.  For CTAs of 256 threads.
template <int BORDER, typename Params>
__device__ __forceinline__ void patch_box_border(float* box, int rows, int bw, int ox, int oy, const Params& p) {
  if (BORDER == KB200_CONSTANT) return;
  if (ox < 0 || oy < 0 || ox + bw > p.W || oy + rows > p.H) {
    for (int e = threadIdx.x; e < rows * bw; e += 256) {
      const int r = e / bw, c = e - r * bw;
      const int gy = oy + r, gx = ox + c;
      if ((unsigned)gy < (unsigned)p.H && (unsigned)gx < (unsigned)p.W) continue;
      const int sr = border_index<BORDER>(gy, p.H) - oy, sc = border_index<BORDER>(gx, p.W) - ox;
      if ((unsigned)sr < (unsigned)rows && (unsigned)sc < (unsigned)bw) box[e] = box[sr * bw + sc];
    }
    __syncthreads();
  }
}

}  // namespace kb200
