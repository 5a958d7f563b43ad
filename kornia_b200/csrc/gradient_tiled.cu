// kornia_b200 -- host dispatch of the tiled image-derivative kernel (gradient_tiled.cuh).
#include "gradient_tiled.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

template <int K, int NOUT, GradEpilogue E>
static int launch_grad_tiled(const CUtensorMap& map, const GradTiledParams& p, cudaStream_t st) {
  constexpr size_t smem = grad_tiled_smem_bytes<K>();
  auto kern = grad_tiled_kernel<K, NOUT, E>;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  KB_SET_SMEM_ONCE(configured, kern, smem);
  kern<<<capped_grid((long long)p.planes * ceil_div(p.H, SEPT_TH), grad_tiled_ctas<K, E>()), 256, smem, st>>>(map, p);
  return launch_status("grad_tiled");
}

// tensor map and parameters shared by every epilogue; false outside the kernel's envelope
static bool grad_tiled_setup(const float* x, const double* taps, float* out, int planes, int H, int W, int nout, int k, CUtensorMap& map,
                             GradTiledParams& p) {
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) return false;
  if (H <= k / 2 || W <= k / 2) return false;
  if ((long long)planes * ceil_div(H, SEPT_TH) > 0x7fffffffll) return false;
  if (!encode_plane_map(&map, x, planes, H, W, SEPT_BW, SEPT_TH + k - 1)) return false;
  p.out = out;
  p.H = H;
  p.W = W;
  p.planes = planes;
  p.eps = 0.f;
  for (int e = 0; e < nout * k * k; ++e) p.taps[e] = (float)taps[e];  // exact: the host built them in fp32
  p.s4 = nullptr;
  p.C = 1;
  return true;
}

int spatial_gradient_tiled_forward(const float* x, const double* taps, float* out, int planes, int H, int W, int nout, int k, int magnitude,
                                   double eps, cudaStream_t st) {
  if (!option(OPT_TILED_GRADIENT) || !option(OPT_TILED_FILTER)) return KB200_EUNSUPPORTED;
  if (!x || !out || !taps || (k != 3 && k != 5) || nout < 2 || nout > GRAD_MAX_OUT) return KB200_EUNSUPPORTED;
  if (magnitude && (nout != 2 || k != 3)) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  GradTiledParams p;
  if (!grad_tiled_setup(x, taps, out, planes, H, W, nout, k, map, p)) return KB200_EUNSUPPORTED;
  p.eps = (float)eps;
  if (magnitude) return launch_grad_tiled<3, 2, GRAD_MAG>(map, p, st);
  if (k == 3 && nout == 2) return launch_grad_tiled<3, 2, GRAD_PLANES>(map, p, st);
  if (k == 3 && nout == 3) return launch_grad_tiled<3, 3, GRAD_PLANES>(map, p, st);
  if (k == 5 && nout == 3) return launch_grad_tiled<5, 3, GRAD_PLANES>(map, p, st);
  return KB200_EUNSUPPORTED;
}

int hessian_tiled_forward(const float* x, const double* taps, const float* s4, float* out, int planes, int C, int H, int W, int k,
                          cudaStream_t st) {
  if (!option(OPT_TILED_GRADIENT) || !option(OPT_TILED_FILTER)) return KB200_EUNSUPPORTED;
  if (!x || !out || !taps || (k != 3 && k != 5)) return KB200_EUNSUPPORTED;
  CUtensorMap map;
  GradTiledParams p;
  if (!grad_tiled_setup(x, taps, out, planes, H, W, 3, k, map, p)) return KB200_EUNSUPPORTED;
  p.s4 = s4;
  p.C = C;
  return k == 3 ? launch_grad_tiled<3, 3, GRAD_HESS>(map, p, st) : launch_grad_tiled<5, 3, GRAD_HESS>(map, p, st);
}

}  // namespace kb200
