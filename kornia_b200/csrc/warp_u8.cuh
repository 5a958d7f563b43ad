// kornia_b200 -- warp straight from the decoder's wire format (SURVEY.md 8f row 4).
//
// An image decoder hands over interleaved uint8 (B,H,W,C).  The reference turns that into the warp's input with two
// full-size passes before the path even starts -- image_to_tensor (kornia/image/utils.py:27: HWC -> CHW permute, made
// contiguous by the first kernel that reads it) and _to_float32 (kornia/io/io.py:108-111: image.float() / 255.0) -- and
// then runs warp_perspective / warp_affine (imgwarp.py:69,177) on the 4x larger fp32 copy.  Here the sampler gathers the
// uint8 taps themselves: C adjacent bytes per tap (the interleaved layout is the better one for a gather: all channels
// of a tap share a 32-byte sector), converts each tap with the rounding of the reference's conversion on this device and
// blends with the very PixelSampler the fp32 kernels use, so the result equals the three-step composition bit for bit.
// Algorithmic bytes per output pixel (C=3): 3 read + 12 written = 15, against 3+12 (ingest) + 12+12 (warp) = 39 for the
// composition on the fp32 kernels of this library, and ~165 for the eager reference.
//
// First version: one thread per output pixel, taps through L1 (the structure of warp_fwd_generic); the shared-memory staged form (byte boxes by TMA: rows of W*C bytes) is the next step.
#pragma once
#include "warp_generic.cuh"

namespace kb200 {

struct WarpU8Params {
  const unsigned char* src;  // (B,H,W,C) interleaved
  const float* m;            // (Bm,3,3)
  const float* bx;           // (w)
  const float* by;           // (h)
  const float* fill;         // (C) or null
  float* out;                // (B,C,h,w) planar
  int B, C, H, W, h, w, Bm, align;
  int normalize;             // value of a byte u: 0 float(u); 1 float(u) * RN(1/255); 2 float(u) / 255 (see below)
  const float* lens;         // undistort only (warp_u8_tiled.cuh, U8_KIND_LENS): (B,16) lens numbers, m / bx / by unused
};

// `image.float() / 255.0` (io.py:111) is evaluated differently by torch's two backends: the CPU kernel divides, the CUDA
// kernel multiplies by the fp32 reciprocal of the scalar (its documented "may lose one bit" shortcut; 126 of the 256 byte
// values differ by one ulp).  normalize=1 is the CUDA form -- what the reference's three steps produce on this device,
// reproduced bit for bit -- and normalize=2 the CPU form.
constexpr float RCP_255 = 0x1.010102p-8f;  // RN(1/255) = 0x3b808081

// float(u) / 255.0f, correctly rounded, without the division: q0 = u * RN(1/255) is off by at most one ulp, one residual
// step repairs it -- e = fma(-255, q0, u) is exact, q = fma(e, r, q0) rounds to the quotient (checked exhaustively over
// the 256 inputs: tools/hostemu and tests/test_ingest_oracle.py).
__device__ __forceinline__ float unit_from_level(float x) {  // x = float(byte)
  const float q0 = __fmul_rn(x, RCP_255);
  const float e = __fmaf_rn(-255.0f, q0, x);
  return __fmaf_rn(e, RCP_255, q0);
}
__device__ __forceinline__ float unit_from_byte(unsigned char u) { return unit_from_level((float)u); }

// value of a tap: one multiply serves normalize 0 (scale 1, exact) and 1 (scale RN(1/255)); 2 takes the residual step
__device__ __forceinline__ float value_of_level(float x, float scale, bool divide) {
  return divide ? unit_from_level(x) : __fmul_rn(x, scale);
}
// float(byte) as 2^23 + byte with the 2^23 removed (one LOP3 + one FADD, both exact) rather than through the conversion pipe
__device__ __forceinline__ float level_of_byte(unsigned char u) { return __fadd_rn(__uint_as_float(0x4B000000u | (unsigned)u), -8388608.0f); }
__device__ __forceinline__ float value_of_byte(unsigned char u, float scale, bool divide) { return value_of_level(level_of_byte(u), scale, divide); }

// float(byte q of word) without the conversion pipe: one PRMT drops the byte into the mantissa of 2^23 (0x4B0000bb =
// 2^23 + bb exactly), one FADD removes the 2^23 -- both exact, so the result is the I2F's.
__device__ __forceinline__ float level_of_word_byte(uint32_t word, int q) {
  return __fadd_rn(__uint_as_float(__byte_perm(word, 0x4B000000u, 0x7540u + (unsigned)q)), -8388608.0f);
}

// NC: channels known at compile time (1 or 3: the loop unrolls, so all C x taps byte loads of a pixel are in flight
// together) or 0 for any p.C.
template <int INTERP, int PAD, int KIND, int NC = 0>
__global__ void __launch_bounds__(GEN_BX* GEN_BY) warp_fwd_u8hwc(const WarpU8Params p) {
  const int x = blockIdx.x * GEN_BX + threadIdx.x;
  const int y = blockIdx.y * GEN_BY + threadIdx.y;
  const int b = blockIdx.z;
  if (x >= p.w || y >= p.h) return;
  Mat3<float> m;
  m.load(p.m + (p.Bm == 1 ? 0 : (size_t)b * 9));
  float gx, gy, den;
  map_point<float, KIND == KIND_PROJ>(m, ldg(p.bx + x), ldg(p.by + y), gx, gy, den);
  const bool align = p.align != 0;
  const int H = p.H, W = p.W, C = NC ? NC : p.C;
  const size_t oplane = (size_t)p.h * p.w;
  const unsigned char* sp = p.src + (size_t)b * H * W * C;
  float* op = p.out + (size_t)b * C * oplane + (size_t)y * p.w + x;
  const float scale = p.normalize == 1 ? RCP_255 : 1.0f;
  const bool divide = p.normalize == 2;

  PixelSampler<float, INTERP, PAD> S;
  S.prepare(unnormalize(gx, W, align), unnormalize(gy, H, align), H, W, align);
#pragma unroll
  for (int ch = 0; ch < C; ++ch) {
    const float v = S.sample_with([&](int off) {
      return value_of_byte(__ldg(sp + (size_t)off * C + ch), scale, divide);
    });
    st_stream(op + ch * oplane, S.finish(v, PAD == KB200_FILL ? ldg(p.fill + ch) : 0.0f));
  }
}

}  // namespace kb200
