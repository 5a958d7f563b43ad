// kornia_b200 -- sub-pixel refinement of 3-D scale-space maxima (conv_quad_interp3d / iterative_quad_interp3d of
// kornia/geometry/subpix/spatial_soft_argmax.py) in one pass per call (fp32).
//
// Every voxel of the (B, C, L, H, W) source gets its grid coordinates [level, x, y] in the contiguous (B, C, 3, L, H, W)
// `coords` and its value in `y`; every maximum of the NMS mask (the given bool mask, or nms3d(x, (3, 3, 3), True)
// computed on the same walk) is then refined by the thread that stored it, so no element is written by two threads.  The refinement is the reference's, in its fp32 operation order with every product and sum rounded on its own:
//  * per iteration, the 3 x 3 x 3 patch at the current position clamped to [1, n - 2] gives g = central differences and
//    the Hessian; H s = -g is solved by Cramer's rule (safe_det = 1 where |det| <= 1e-7f: unsolved);
//  * the conv form also needs the reference's table hit: some mask-True voxel of the same volume within L-inf distance
//    `radius` of the clamped position (always true within `radius` of the keypoint's own maximum);
//  * an unsolved (or missed) keypoint stops with its last shift; a solved one takes the shift and moves one step along
//    x, then y, then (allow_scale) the level where |shift| > max_shift, each move checked against [1, n - 2] and the
//    position then clamped to [0, n - 1];
//  * at the end, valid = still valid and |shift| <= 1.5 on all axes: coords = position + shift, else the grid;
//    y = x[position] + 0.5 * (valid ? g . s : 0) (+ bonus * valid when the bonus is > 0).
// An iteration that leaves a valid keypoint where it was repeats itself, so the loop stops there: the result is the
// n_iters-iteration result.  A NaN in a patch makes det NaN and the keypoint unsolved.
//
// Walk: persistent CTAs over 128 x 8 tiles of one (b, c) volume walk the level axis with nms.cuh's staging and
// three-level ring (without a mask), or stream the given mask (with one).  Each thread owns 4 adjacent columns and stores
// them as float4 where aligned.  Patches are read with __ldg from the L2-resident source, because a keypoint can walk off
// its tile.  The source's H x W planes are dense; its b, c and level strides are arguments, so a permuted view is read in
// place; `y` is written at its own strides (those of input.clone()).
//
// Launched by quad_interp.cu; tests/test_subpix_gpu.py checks it bit for bit against the composition, and tools/hostemu
// (run_emu --quad) runs it on the host against a scalar restatement.
#pragma once
#include "nms.cuh"

namespace kb200 {

struct QuadParams {
  const float* src;            // (B, C, L, H, W) with dense H x W planes at sB, sC, sL
  const unsigned char* mask;   // contiguous (B, C, L, H, W) bool, or null: the NMS mask is computed on the walk
  float* coords;               // contiguous (B, C, 3, L, H, W)
  float* y;                    // (B, C, L, H, W) at ysB, ysC, ysL, ysH, ysW
  long long sB, sC, sL;
  long long ysB, ysC, ysL, ysH, ysW;
  int C, L, H, W, tiles_x, tiles_y;
  long long tiles;             // vols * tiles_y * tiles_x
  int n_iters, radius;         // radius: the conv form's dilation radius (>= 1); unused by the iterative form
  float max_shift, bonus;      // the Python floats rounded to fp32, as torch compares and adds them
  int add_bonus, allow_scale;  // add_bonus: strict_maxima_bonus > 0
  int refine;                  // 0 when L, H or W < 3: the grid and the copy only
};

// nms3d(x, (3, 3, 3), True) at one voxel, from global memory: strictly above the NaN-propagating max of its 26
// neighbours, False on the border.
__device__ __forceinline__ bool quad_strict_max(const float* vol, const QuadParams& p, int d, int h, int w) {
  if (d < 1 || d > p.L - 2 || h < 1 || h > p.H - 2 || w < 1 || w > p.W - 2) return false;
  const float* c = vol + d * p.sL + h * p.W + w;
  float m = ldg(c - p.sL - p.W - 1);
  for (int dd = -1; dd <= 1; ++dd)
    for (int dh = -1; dh <= 1; ++dh)
      for (int dw = -1; dw <= 1; ++dw)
        if (dd || dh || dw) m = nan_max(m, ldg(c + dd * p.sL + dh * p.W + dw));
  return ldg(c) > m;
}

// The conv form's table lookup at the clamped position (d, h, w) of a keypoint whose maximum is at (d0, h0, w0).
template <bool HAS_MASK>
__device__ bool quad_table_hit(const float* vol, const unsigned char* mvol, const QuadParams& p, int d, int h, int w, int d0, int h0, int w0) {
  const int r = p.radius;
  if (abs(d - d0) <= r && abs(h - h0) <= r && abs(w - w0) <= r) return true;  // the keypoint's own maximum
  for (int dd = max(d - r, 0); dd <= min(d + r, p.L - 1); ++dd)
    for (int hh = max(h - r, 0); hh <= min(h + r, p.H - 1); ++hh)
      for (int ww = max(w - r, 0); ww <= min(w + r, p.W - 1); ++ww) {
        const bool m = HAS_MASK ? mvol[((long long)dd * p.H + hh) * p.W + ww] != 0 : quad_strict_max(vol, p, dd, hh, ww);
        if (m) return true;
      }
  return false;
}

// Refine the maximum at (d0, h0, w0): out = {level, x, y, value}.
template <bool HAS_MASK, bool CONV>
__device__ void quad_refine(const float* vol, const unsigned char* mvol, const QuadParams& p, int d0, int h0, int w0, float out[4]) {
  using R = RN<float>;
  int d = d0, h = h0, w = w0;
  bool valid = true;
  float shx = 0.f, shy = 0.f, shs = 0.f, gds = 0.f;
  for (int it = 0; it < p.n_iters; ++it) {
    const int di = min(max(d, 1), p.L - 2), hi = min(max(h, 1), p.H - 2), wi = min(max(w, 1), p.W - 2);
    const float* c = vol + di * p.sL + hi * p.W + wi;
    const long long sL = p.sL, sH = p.W;
    auto at = [&](int dd, int dh, int dw) { return ldg(c + dd * sL + dh * sH + dw); };
    const float cc = at(0, 0, 0), xm = at(0, 0, -1), xp = at(0, 0, 1), ym = at(0, -1, 0), yp = at(0, 1, 0), sm = at(-1, 0, 0), sp = at(1, 0, 0);
    const float gx = R::mul(0.5f, R::sub(xp, xm)), gy = R::mul(0.5f, R::sub(yp, ym)), gs = R::mul(0.5f, R::sub(sp, sm));
    const float c2 = R::mul(2.f, cc);
    const float dxx = R::add(R::sub(xp, c2), xm), dyy = R::add(R::sub(yp, c2), ym), dss = R::add(R::sub(sp, c2), sm);
    const float dxy = R::mul(0.25f, R::add(R::sub(R::sub(at(0, 1, 1), at(0, 1, -1)), at(0, -1, 1)), at(0, -1, -1)));
    const float dxs = R::mul(0.25f, R::add(R::sub(R::sub(at(1, 0, 1), at(1, 0, -1)), at(-1, 0, 1)), at(-1, 0, -1)));
    const float dys = R::mul(0.25f, R::add(R::sub(R::sub(at(1, 1, 0), at(1, -1, 0)), at(-1, 1, 0)), at(-1, -1, 0)));
    // _solve_cramer_sym3x3(dxx, dyy, dss, dxy, dxs, dys, -gx, -gy, -gs)
    const float r0 = -gx, r1 = -gy, r2 = -gs;
    const float cf00 = R::sub(R::mul(dyy, dss), R::mul(dys, dys));
    const float cf01 = R::sub(R::mul(dxy, dss), R::mul(dys, dxs));
    const float cf02 = R::sub(R::mul(dxy, dys), R::mul(dyy, dxs));
    const float det = R::add(R::sub(R::mul(dxx, cf00), R::mul(dxy, cf01)), R::mul(dxs, cf02));
    bool ok = fabsf(det) > 1e-7f;
    const float sd = ok ? det : 1.f;
    const float t1 = R::sub(R::mul(r1, dss), R::mul(dys, r2)), t2 = R::sub(R::mul(r1, dys), R::mul(dyy, r2));
    const float t3 = R::sub(R::mul(dxy, r2), R::mul(r1, dxs)), t4 = R::sub(R::mul(dyy, r2), R::mul(r1, dys));
    const float sx = R::div(R::add(R::sub(R::mul(r0, cf00), R::mul(dxy, t1)), R::mul(dxs, t2)), sd);
    const float sy = R::div(R::add(R::sub(R::mul(dxx, t1), R::mul(r0, cf01)), R::mul(dxs, t3)), sd);
    const float ss = R::div(R::add(R::sub(R::mul(dxx, t4), R::mul(dxy, t3)), R::mul(r0, cf02)), sd);
    if (CONV) ok = ok && quad_table_hit<HAS_MASK>(vol, mvol, p, di, hi, wi, d0, h0, w0);
    if (!ok) {  // invalid from here on: the shift and the position stay what they were
      valid = false;
      break;
    }
    shx = sx;
    shy = sy;
    shs = ss;
    gds = R::add(R::add(R::mul(gx, sx), R::mul(gy, sy)), R::mul(gs, ss));
    const int d_in = d, h_in = h, w_in = w;
    const int nw = w + (sx > p.max_shift) - (sx < -p.max_shift);
    valid = nw >= 1 && nw <= p.W - 2;
    w = min(max(nw, 0), p.W - 1);
    if (valid) {
      const int nh = h + (sy > p.max_shift) - (sy < -p.max_shift);
      valid = nh >= 1 && nh <= p.H - 2;
      h = min(max(nh, 0), p.H - 1);
    }
    if (valid && p.allow_scale) {
      const int nd = d + (ss > p.max_shift) - (ss < -p.max_shift);
      valid = nd >= 1 && nd <= p.L - 2;
      d = min(max(nd, 0), p.L - 1);
    }
    if (!valid || (d == d_in && h == h_in && w == w_in)) break;  // frozen, or the next iteration repeats this one
  }
  valid = valid && fabsf(shx) <= 1.5f && fabsf(shy) <= 1.5f && fabsf(shs) <= 1.5f;
  out[0] = valid ? R::add((float)d, shs) : (float)d0;
  out[1] = valid ? R::add((float)w, shx) : (float)w0;
  out[2] = valid ? R::add((float)h, shy) : (float)h0;
  float v = R::add(ldg(vol + d * p.sL + h * p.W + w), R::mul(0.5f, valid ? gds : 0.f));
  if (p.add_bonus) v = R::add(v, R::mul(p.bonus, valid ? 1.f : 0.f));
  out[3] = v;
}

// Four adjacent values of one row: a float4 when the group lies in the row, the column stride is 1 and the address is
// aligned, else one by one.
__device__ __forceinline__ void quad_store4(float* o, long long sw, int gx, int W, const float v[4]) {
  if (gx + 3 < W && sw == 1 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
    *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (gx + i < W) o[i * sw] = v[i];
  }
}

template <bool HAS_MASK, bool CONV>
__global__ void __launch_bounds__(NMS3_NT) quad_interp3d_kernel(const QuadParams p) {
  extern __shared__ __align__(128) unsigned char nms_smem[];
  float* s = reinterpret_cast<float*>(nms_smem);
  const int tid = threadIdx.x;
  const int c4 = (tid & 31) * 4, ry = tid >> 5;
  const long long HW = (long long)p.H * p.W;
  for (long long t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    const int tx = (int)(t % p.tiles_x);
    const long long rest = t / p.tiles_x;
    const int ty = (int)(rest % p.tiles_y);
    const int vol = (int)(rest / p.tiles_y);
    const int x0 = tx * NMS3_TW, y0 = ty * NMS3_TH;
    const int gy = y0 + ry, gx = x0 + c4;
    const bool active = gy < p.H && gx < p.W;
    const bool row_in = gy >= 1 && gy < p.H - 1;
    const int b = vol / p.C, ch = vol % p.C;
    const float* src = p.src + (long long)b * p.sB + (long long)ch * p.sC;
    const unsigned char* mvol = HAS_MASK ? p.mask + (long long)vol * p.L * HW : nullptr;
    // without a mask, the ring of nms3d_kernel: 3 x 3 max of level l - 2, and of level l - 1 its centre, 3 x 3 and
    // 8-neighbour max; level l - 1 is emitted once level l is staged
    float pmax[4] = {}, cmax[4] = {}, c8max[4] = {}, cval[4] = {};
    for (int l = 0; l < p.L + (HAS_MASK ? 0 : 1); ++l) {
      float nmax[4] = {}, n8max[4] = {}, nval[4] = {}, unused[4];
      if (!HAS_MASK && l < p.L) nms3_stage_level<false>(s, src + (long long)l * p.sL, p.H, p.W, x0, y0, tid, c4, ry, nval, nmax, n8max, unused, unused);
      const int e = HAS_MASK ? l : l - 1;
      if (e >= 0 && active) {
        float xv[4];
        bool keep[4];
        if (HAS_MASK) {
          const float* row = src + (long long)e * p.sL + (long long)gy * p.W + gx;
          const unsigned char* mrow = mvol + ((long long)e * p.H + gy) * p.W + gx;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            xv[i] = gx + i < p.W ? ldg(row + i) : 0.f;
            keep[i] = p.refine && gx + i < p.W && mrow[i] != 0;
          }
        } else {
          const bool level_in = p.refine && l >= 2 && l < p.L && row_in;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            xv[i] = cval[i];
            keep[i] = level_in && gx + i >= 1 && gx + i < p.W - 1 && nms3_is_max(cval[i], pmax[i], c8max[i], nmax[i]);
          }
        }
        float cs[4], cx[4], cy[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          cs[i] = (float)e;
          cx[i] = (float)(gx + i);
          cy[i] = (float)gy;
        }
        const long long co = (((long long)vol * 3 * p.L + e) * p.H + gy) * p.W + gx, cstep = (long long)p.L * HW;
        float* yo = p.y + b * p.ysB + ch * p.ysC + e * p.ysL + gy * p.ysH + gx * p.ysW;
        quad_store4(p.coords + co, 1, gx, p.W, cs);
        quad_store4(p.coords + co + cstep, 1, gx, p.W, cx);
        quad_store4(p.coords + co + 2 * cstep, 1, gx, p.W, cy);
        quad_store4(yo, p.ysW, gx, p.W, xv);
        // the maxima (about 0.1 - 1 % of the voxels) overwrite what this thread just stored: one call site, not unrolled
        int todo = (keep[0] ? 1 : 0) | (keep[1] ? 2 : 0) | (keep[2] ? 4 : 0) | (keep[3] ? 8 : 0);
        while (todo) {
          const int i = __ffs(todo) - 1;
          todo &= todo - 1;
          float r[4];
          quad_refine<HAS_MASK, CONV>(src, mvol, p, e, gy, gx + i, r);
          p.coords[co + i] = r[0];
          p.coords[co + cstep + i] = r[1];
          p.coords[co + 2 * cstep + i] = r[2];
          yo[i * p.ysW] = r[3];
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        pmax[i] = cmax[i];
        cmax[i] = nmax[i];
        c8max[i] = n8max[i];
        cval[i] = nval[i];
      }
    }
  }
}

int quad_interp3d_forward(const float* x, const unsigned char* mask, float* coords, float* y, int B, int C, int L, int H, int W,
                          long long sB, long long sC, long long sL, long long ysB, long long ysC, long long ysL, long long ysH,
                          long long ysW, int n_iters, int radius, float max_shift, float bonus, int add_bonus, int allow_scale, cudaStream_t st);

}  // namespace kb200
