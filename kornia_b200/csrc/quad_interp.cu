// kornia_b200 -- host side of the sub-pixel refinement kernel (quad_interp.cuh).
#include "persistent_launch.cuh"
#include "quad_interp.cuh"

namespace kb200 {

template <bool HAS_MASK, bool CONV>
static int launch_quad(const QuadParams& p, cudaStream_t st) {
  auto kern = quad_interp3d_kernel<HAS_MASK, CONV>;
  const int smem = HAS_MASK ? 0 : NMS3_SMEM_BYTES;  // the NMS walk stages each level; a given mask is streamed
  kern<<<persistent_grid(kern, NMS3_NT, smem, p.tiles), NMS3_NT, smem, st>>>(p);
  return launch_status("quad_interp3d_kernel");
}

int quad_interp3d_forward(const float* x, const unsigned char* mask, float* coords, float* y, int B, int C, int L, int H, int W,
                          long long sB, long long sC, long long sL, long long ysB, long long ysC, long long ysL, long long ysH,
                          long long ysW, int n_iters, int radius, float max_shift, float bonus, int add_bonus, int allow_scale, cudaStream_t st) {
  QuadParams p{};
  p.src = x;
  p.mask = mask;
  p.coords = coords;
  p.y = y;
  p.sB = sB;
  p.sC = sC;
  p.sL = sL;
  p.ysB = ysB;
  p.ysC = ysC;
  p.ysL = ysL;
  p.ysH = ysH;
  p.ysW = ysW;
  p.C = C;
  p.L = L;
  p.H = H;
  p.W = W;
  p.tiles_x = ceil_div(W, NMS3_TW);
  p.tiles_y = ceil_div(H, NMS3_TH);
  p.tiles = (long long)B * C * p.tiles_y * p.tiles_x;
  p.n_iters = n_iters;
  // a radius past the volume's largest side reaches every voxel either way; the clamp keeps d +- r in int range
  const int side = max(L, max(H, W));
  p.radius = radius < side ? radius : side;
  p.max_shift = max_shift;
  p.bonus = bonus;
  p.add_bonus = add_bonus != 0;
  p.allow_scale = allow_scale != 0;
  p.refine = L >= 3 && H >= 3 && W >= 3;
  const bool conv = radius > 0;
  if (mask) return conv ? launch_quad<true, true>(p, st) : launch_quad<true, false>(p, st);
  return conv ? launch_quad<false, true>(p, st) : launch_quad<false, false>(p, st);
}

}  // namespace kb200
