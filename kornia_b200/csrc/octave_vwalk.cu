// kornia_b200 -- host side of the ScalePyramid octave kernel (octave_vwalk.cuh).
#include "octave_vwalk.cuh"
#include "persistent_launch.cuh"

namespace kb200 {

template <typename CH>
static int launch_octave(const OctaveParams& p, cudaStream_t st) {
  auto kern = octave_vwalk_kernel<CH>;
  static unsigned long long configured = 0;
  KB_SET_SMEM_ONCE(configured, kern, CH::SMEM_BYTES());
  const long long strips = (long long)p.planes * ceil_div(p.W, OCT_BW);
  const long long steps = ceil_div(p.H + CH::D(CH::L - 1), OCT_TH);
  // segments of at least 3 PRIME steps, so a segment that starts inside a band spends at most a quarter of its steps refilling
  const long long want = strips * steps / (3 * CH::PRIME() > 0 ? 3 * CH::PRIME() : 1);
  kern<<<capped_grid(want < 1 ? 1 : want, 1), OCT_NT, CH::SMEM_BYTES(), st>>>(p);
  return launch_status("octave_vwalk");
}

template <typename CH>
static bool chain_is(const int* ksizes, int L) {
  if (L != CH::L || (ksizes[0] > 0) != CH::BLUR0) return false;
  for (int l = CH::BLUR0 ? 0 : 1; l < L; ++l)
    if (ksizes[l] != CH::K[l]) return false;
  return true;
}

// the chains of ScalePyramid() (11..25 from init 13), ScaleSpaceDetector's ScalePyramid(3, 1.6, 16, extra_levels=2)
// (11..21 from init 13) and the double_image pyramid of SIFTFeature / HesAffNetHardNet / GFTTAffNetHardNet (11..25 from
// init 11), each with a copy stage for the later octaves
using OctDefault = OctaveChain<13, 11, 13, 17, 21, 25>;
using OctDetector = OctaveChain<13, 11, 13, 17, 21>;
using OctDouble = OctaveChain<11, 11, 13, 17, 21, 25>;
using OctCopy6 = OctaveChain<0, 11, 13, 17, 21, 25>;
using OctCopy5 = OctaveChain<0, 11, 13, 17, 21>;

int octave_vwalk_forward(const float* x, const double* taps, const int* ksizes, int L, float* out, int planes, int H, int W, cudaStream_t st) {
  if (L < 2 || L > OCT_MAX_L) return KB200_EUNSUPPORTED;
  for (int l = 0; l < L; ++l)
    if (ksizes[l] > H || ksizes[l] > W) return KB200_EUNSUPPORTED;  // the reference blurs such a level with gaussian_blur2d
  if ((W % 4) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) return KB200_EUNSUPPORTED;
  if ((long long)planes * ceil_div(W, OCT_BW) > 0x7fffffffll) return KB200_EUNSUPPORTED;
  OctaveParams p{};
  p.src = x;
  p.out = out;
  p.planes = planes;
  p.H = H;
  p.W = W;
  int off = 0;
  for (int l = 0; l < L; ++l) {
    if (ksizes[l] > OCT_MAX_K) return KB200_EUNSUPPORTED;
    for (int j = 0; j < ksizes[l]; ++j) p.taps[l][j] = (float)taps[off + j];  // exact: fp32 taps
    off += ksizes[l];
  }
  if (chain_is<OctDefault>(ksizes, L)) return launch_octave<OctDefault>(p, st);
  if (chain_is<OctDetector>(ksizes, L)) return launch_octave<OctDetector>(p, st);
  if (chain_is<OctDouble>(ksizes, L)) return launch_octave<OctDouble>(p, st);
  if (chain_is<OctCopy6>(ksizes, L)) return launch_octave<OctCopy6>(p, st);
  if (chain_is<OctCopy5>(ksizes, L)) return launch_octave<OctCopy5>(p, st);
  return KB200_EUNSUPPORTED;
}

}  // namespace kb200
