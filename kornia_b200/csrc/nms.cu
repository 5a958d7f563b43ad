// kornia_b200 -- host side of the non-maximum-suppression kernels (nms.cuh).
#include "nms.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

template <int K, bool VALUES>
static int launch_nms2d(const Nms2dParams& p, cudaStream_t st) {
  auto kern = nms2d_kernel<K, VALUES>;
  constexpr int smem = Nms2dShape<K>::BYTES;
  static_assert(smem <= 48 * 1024, "the 2-D tile must fit the default shared-memory limit");
  kern<<<persistent_grid(kern, NMS_NT, smem, p.tiles), NMS_NT, smem, st>>>(p);
  return launch_status("nms2d_kernel");
}

template <bool VALUES>
static int dispatch_nms2d(const Nms2dParams& p, int k, cudaStream_t st) {
  switch (k) {
    case 3: return launch_nms2d<3, VALUES>(p, st);
    case 5: return launch_nms2d<5, VALUES>(p, st);
    case 7: return launch_nms2d<7, VALUES>(p, st);
    case 9: return launch_nms2d<9, VALUES>(p, st);
    case 11: return launch_nms2d<11, VALUES>(p, st);
    case 13: return launch_nms2d<13, VALUES>(p, st);
    case 15: return launch_nms2d<15, VALUES>(p, st);
    case 17: return launch_nms2d<17, VALUES>(p, st);
    case 19: return launch_nms2d<19, VALUES>(p, st);
    case 21: return launch_nms2d<21, VALUES>(p, st);
    case 23: return launch_nms2d<23, VALUES>(p, st);
    case 25: return launch_nms2d<25, VALUES>(p, st);
    case 27: return launch_nms2d<27, VALUES>(p, st);
    case 29: return launch_nms2d<29, VALUES>(p, st);
    case 31: return launch_nms2d<31, VALUES>(p, st);
    default: return KB200_EUNSUPPORTED;
  }
}

int nms2d_forward(const float* x, void* out, int B, int C, int H, int W, long long sB, long long sC, int k, bool values, cudaStream_t st) {
  if (k < 3 || k > 31 || k % 2 == 0) return KB200_EUNSUPPORTED;
  Nms2dParams p{};
  p.src = x;
  p.out = out;
  p.sB = sB;
  p.sC = sC;
  p.C = C;
  p.H = H;
  p.W = W;
  p.tiles_x = ceil_div(W, NMS_TW);
  p.tiles_y = ceil_div(H, NMS_TH);
  p.tiles = (long long)B * C * p.tiles_y * p.tiles_x;
  return values ? dispatch_nms2d<true>(p, k, st) : dispatch_nms2d<false>(p, k, st);
}

template <int MODE>
static int launch_nms3d(const Nms3dParams& p, cudaStream_t st) {
  auto kern = nms3d_kernel<MODE>;
  kern<<<persistent_grid(kern, NMS3_NT, NMS3_SMEM_BYTES, p.tiles), NMS3_NT, NMS3_SMEM_BYTES, st>>>(p);
  return launch_status("nms3d_kernel");
}

int nms3d_forward(const float* x, void* out0, void* out1, int B, int C, int L, int H, int W, long long sB, long long sC, long long sL,
                  int mode, cudaStream_t st) {
  Nms3dParams p{};
  p.src = x;
  p.out0 = out0;
  p.out1 = out1;
  p.sB = sB;
  p.sC = sC;
  p.sL = sL;
  p.C = C;
  p.L = L;
  p.H = H;
  p.W = W;
  p.tiles_x = ceil_div(W, NMS3_TW);
  p.tiles_y = ceil_div(H, NMS3_TH);
  p.tiles = (long long)B * C * p.tiles_y * p.tiles_x;
  switch (mode) {
    case NMS3_MAX_MASK: return launch_nms3d<NMS3_MAX_MASK>(p, st);
    case NMS3_MAX_VALUES: return launch_nms3d<NMS3_MAX_VALUES>(p, st);
    case NMS3_MINMAX: return launch_nms3d<NMS3_MINMAX>(p, st);
    default: return KB200_EUNSUPPORTED;
  }
}

}  // namespace kb200
