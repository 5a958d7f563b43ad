// kornia_b200 -- coordinate transforms of the sampler (device).
//
// Semantics: ATen grid_sampler_2d as called by the reference at
// kornia/geometry/transform/imgwarp.py:174,290,316,320,702.  Spec followed:
// torch/include/ATen/native/GridSampler.h:27-35 (unnormalise), :58-60 (clip), :89-105 (reflect),
// :143-160 (compute_coordinates), UpSample.h:398-423 (cubic convolution, A = -0.75), and the
// CUDA flavour's non-finite guard (cuda/GridSampler.cuh: out-of-int-range / NaN -> -100).
#pragma once
#include "common.cuh"

namespace kb200 {

template <typename T>
__device__ __forceinline__ T unnormalize(T g, int size, bool align) {
  using R = RN<T>;
  if (align) return R::mul(R::mul(R::add(g, T(1)), T(0.5)), T(size - 1));
  // ((g + 1) * size - 1) / 2 as ATen's CUDA kernel evaluates it: nvcc contracts the product and the subtraction into one FMA
  // there (cuda/GridSampler.cuh is built with -fmad=true), so the same-device reference is reproduced bit for bit
  // (tests/test_parity_gpu.py::test_warp_forward_fp32_equals_the_same_device_reference); torch's CPU kernel rounds the product
  // separately -- a one-ulp difference in the coordinate, inside the reference's own CPU-vs-CUDA gap.
  return R::mul(R::fma(R::add(g, T(1)), T(size), T(-1)), T(0.5));
}

template <typename T>
__device__ __forceinline__ T clip_coord(T c, int size) {
  return fmin(T(size - 1), fmax(c, T(0)));
}

template <typename T>
__device__ __forceinline__ T reflect_coord(T c, int twice_low, int twice_high) {
  using R = RN<T>;
  if (twice_low == twice_high) return T(0);
  const T lo = T(twice_low) * T(0.5);
  const T span = T(twice_high - twice_low) * T(0.5);
  c = R::abs(R::sub(c, lo));
  const T extra = R::fmod(c, span);
  const int flips = static_cast<int>(R::floor(R::div(c, span)));
  return (flips % 2 == 0) ? R::add(extra, lo) : R::add(R::sub(span, extra), lo);
}

// Inside the image the reflection of GridSampler.h:89-105 is the identity -- up to its own rounding: with align_corners=False
// the coordinate makes a round trip through the half-pixel offset (|c - (-0.5)|, fmod by the span, + (-0.5)).  The tiled
// kernels restrict their fast path to interior pixels under 'reflection' and apply exactly this round trip there, so that they
// agree with reflect_coord (and with ATen) bit for bit.
template <int PAD, bool ALIGN>
__device__ __forceinline__ float interior_reflection(float c) {
  if (PAD == KB200_REFLECTION && !ALIGN) return RN<float>::add(RN<float>::sub(c, -0.5f), -0.5f);
  return c;
}

// reflect_coord + clip_coord ('reflection' of a bilinear / nearest coordinate, GridSampler.h:89-105,143-160) as straight-line
// code for coordinates within one span of the image -- which is every pixel of a border tile: |c - lo| < span has flips = 0 and
// fmod = identity, span <= |c - lo| < 2 span has flips = 1 and fmod(a, span) = a - span EXACTLY (Sterbenz).  Anything further out
// (or NaN) raises `far` and the caller sends the pixel to its exact path, where reflect_coord itself runs.  Bit-identical to
// clip_coord(reflect_coord(...)) wherever `far` stays false (tools/hostemu checks it).
// (With the general reflect_coord inlined as a third branch here, the border tiles of a 1080p warp cost several interior tiles.)
template <typename T>
__device__ __forceinline__ T reflect_clip_near_rt(T c, int size, bool align, bool& far) {
  using R = RN<T>;
  if (align) {
    // lo = 0, span = size - 1: c - 0 and e + 0 are the identity (e >= +0) and the reflected value already lies in [0, size - 1],
    // so the clip is one too -- the general form below minus its four no-ops (16 -> 7 instructions per coordinate, paid
    // 32 times per pixel quad by the 'reflection' remap)
    if (size == 1) return T(0);  // a one-texel axis (uniform)
    const T span = T(size - 1);
    const T a = R::abs(c);
    far = far || !(a < T(2) * span);
    return a < span ? a : R::sub(span, R::sub(a, span));
  }
  const T lo = T(-0.5), span = T(size);
  const T a = R::abs(R::sub(c, lo));
  far = far || !(a < T(2) * span);
  const T e = a < span ? a : R::sub(span, R::sub(a, span));
  return clip_coord(R::add(e, lo), size);
}
template <bool ALIGN>
__device__ __forceinline__ float reflect_clip_near(float c, int size, bool& far) {
  return reflect_clip_near_rt<float>(c, size, ALIGN, far);
}

// values that cannot be an index (NaN, +-inf, beyond int range) become -100: out of bounds
template <typename T>
__device__ __forceinline__ T guard_index(T c) {
  return (RN<T>::abs(c) <= T(2147483648.0)) ? c : T(-100);
}

template <typename T, int PAD>
__device__ __forceinline__ T pad_coord(T c, int size, bool align) {
  if (PAD == KB200_BORDER) {
    c = clip_coord(c, size);
  } else if (PAD == KB200_REFLECTION) {
    // within one span of the image (all but pathological maps) the reflection is two subtractions and a select; only beyond that
    // the general form with fmod / division runs.  Both agree bit for bit where the first applies.  (With the
    // general form alone, the exact-path pixels of ONE badly fitting sample make its CTAs stragglers.)
    bool far = false;
    const T near = reflect_clip_near_rt<T>(c, size, align, far);
    c = far ? clip_coord(align ? reflect_coord(c, 0, 2 * (size - 1)) : reflect_coord(c, -1, 2 * size - 1), size) : near;
  }
  return guard_index(c);
}

// Same, also returning d(out)/d(in) (GridSampler.h:176-203): borders count as out of bounds.
template <typename T, int PAD>
__device__ __forceinline__ T pad_coord_grad(T c, int size, bool align, T* mult) {
  using R = RN<T>;
  T g = T(1);
  if (PAD == KB200_REFLECTION) {
    const int tl = align ? 0 : -1;
    const int th = align ? 2 * (size - 1) : 2 * size - 1;
    if (tl == th) {
      c = T(0);
      g = T(0);
    } else {
      const T lo = T(tl) * T(0.5);
      const T span = T(th - tl) * T(0.5);
      c = R::sub(c, lo);
      T sgn = T(1);
      if (c < T(0)) {
        sgn = T(-1);
        c = -c;
      }
      const T extra = R::fmod(c, span);
      const int flips = static_cast<int>(R::floor(R::div(c, span)));
      if (flips % 2 == 0) {
        c = R::add(extra, lo);
        g = sgn;
      } else {
        c = R::add(R::sub(span, extra), lo);
        g = -sgn;
      }
    }
  }
  if (PAD == KB200_BORDER || PAD == KB200_REFLECTION) {
    const T hi = T(size - 1);
    if (c <= T(0)) {
      c = T(0);
      g = T(0);
    } else if (c >= hi) {
      c = hi;
      g = T(0);
    }
  }
  *mult = g;
  return guard_index(c);
}

// cubic convolution weights for the four taps at offsets -1, 0, 1, 2 (A = -0.75), Horner form with the
// fused multiply-adds a -fmad=true build of UpSample.h:398-423 produces (explicit, so every kernel of
// this library rounds them identically)
template <typename T>
__device__ __forceinline__ void cubic_weights(T t, T w[4]) {
  using R = RN<T>;
  const T A = T(-0.75);
  const T x0 = R::add(t, T(1));
  w[0] = R::fma(R::fma(R::fma(A, x0, T(3.75)), x0, T(-6)), x0, T(3));          // ((A x - 5A) x + 8A) x - 4A
  w[1] = R::fma(R::mul(R::fma(T(1.25), t, T(-2.25)), t), t, T(1));             // ((A+2) x - (A+3)) x x + 1
  const T u = R::sub(T(1), t);
  w[2] = R::fma(R::mul(R::fma(T(1.25), u, T(-2.25)), u), u, T(1));
  const T x3 = R::add(u, T(1));
  w[3] = R::fma(R::fma(R::fma(A, x3, T(3.75)), x3, T(-6)), x3, T(3));
}

// d(weights)/dt (GridSampler.h get_cubic_coefficients_grad)
template <typename T>
__device__ __forceinline__ void cubic_weights_grad(T t, T w[4]) {
  const T A = T(-0.75);
  T x = T(-1) - t;
  w[0] = (T(-3) * A * x - T(10) * A) * x - T(8) * A;
  x = -t;
  w[1] = (T(-3) * (A + T(2)) * x - T(2) * (A + T(3))) * x;
  x = T(1) - t;
  w[2] = (T(3) * (A + T(2)) * x - T(2) * (A + T(3))) * x;
  x = T(2) - t;
  w[3] = (T(3) * A * x - T(10) * A) * x + T(8) * A;
}

__device__ __forceinline__ bool in_bounds(int y, int x, int H, int W) {
  return (unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W;
}

// Exact per-pixel sampler on a global-memory plane: everything about one output pixel that does not
// depend on the channel (tap offsets, bounds flags, weights, fill coverage) is prepared once, then
// `sample(plane)` is called per channel.  Shared by the generic kernel and by the careful path of the
// tiled kernel, so the two are the same arithmetic by construction.  PAD == KB200_FILL samples with
// zeros padding and exposes 1 - coverage (imgwarp.py:308-320).
template <typename T, int INTERP, int PAD>
struct PixelSampler {
  static constexpr int SPAD = (PAD == KB200_FILL) ? KB200_ZEROS : PAD;
  static constexpr int NT = (INTERP == KB200_BICUBIC) ? 4 : 1;
  int o;            // bilinear / nearest: offset of the first tap
  int W;
  bool ok[4];       // bilinear: nw, ne, sw, se ; nearest: ok[0]
  T w[4];           // bilinear weights
  int xo[NT], yo[NT];
  bool xok[NT], yok[NT];
  T cx[NT], cy[NT];
  T inv_cover;

  __device__ __forceinline__ void prepare(T ix, T iy, int H, int W_, bool align) { prepare_rows(ix, iy, H, W_, W_, align); }

  // Same, on a plane whose rows lie `row` elements apart (row >= W_): bounds and padding use the width W_, tap offsets the row
  // stride.  prepare() is the contiguous case, row == W_.
  __device__ __forceinline__ void prepare_rows(T ix, T iy, int H, int W_, int row, bool align) {
    using R = RN<T>;
    W = row;
    inv_cover = T(0);
    if (INTERP == KB200_BILINEAR) {
      ix = pad_coord<T, SPAD>(ix, W_, align);
      iy = pad_coord<T, SPAD>(iy, H, align);
      const T x0f = R::floor(ix), y0f = R::floor(iy);
      const T x1f = R::add(x0f, T(1)), y1f = R::add(y0f, T(1));
      const T wx1 = R::sub(x1f, ix), wx0 = R::sub(ix, x0f);
      const T wy1 = R::sub(y1f, iy), wy0 = R::sub(iy, y0f);
      w[0] = R::mul(wx1, wy1); w[1] = R::mul(wx0, wy1); w[2] = R::mul(wx1, wy0); w[3] = R::mul(wx0, wy0);
      const int x0 = (int)x0f, y0 = (int)y0f;
      ok[0] = in_bounds(y0, x0, H, W_); ok[1] = in_bounds(y0, x0 + 1, H, W_);
      ok[2] = in_bounds(y0 + 1, x0, H, W_); ok[3] = in_bounds(y0 + 1, x0 + 1, H, W_);
      o = y0 * W + x0;
      if (PAD == KB200_FILL) {
        T cover = T(0);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (ok[k]) cover = R::add(cover, w[k]);
        inv_cover = R::sub(T(1), cover);
      }
    } else if (INTERP == KB200_NEAREST) {
      ix = pad_coord<T, SPAD>(ix, W_, align);
      iy = pad_coord<T, SPAD>(iy, H, align);
      const int xn = (int)R::rint(ix), yn = (int)R::rint(iy);
      ok[0] = in_bounds(yn, xn, H, W_);
      o = yn * W + xn;
      if (PAD == KB200_FILL) inv_cover = ok[0] ? T(0) : T(1);
    } else {  // bicubic: coordinates stay un-padded, every tap is padded on its own
      const T fx = R::floor(ix), fy = R::floor(iy);
      cubic_weights<T>(R::sub(ix, fx), cx);
      cubic_weights<T>(R::sub(iy, fy), cy);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        // the tap coordinates as ATen's forward spells them: ix_nw - 1, ix_nw + 0, ix_nw + 1, ix_nw + 2 but iy_nw - 1 + i.  The
        // same values below 2^24; beyond it (fx - 1) + 2 and fx + 1 round differently, which 'reflection' folds to other texels.
        const int xi = (int)pad_coord<T, SPAD>(R::add(fx, T(i - 1)), W_, align);
        const int yi = (int)pad_coord<T, SPAD>(R::add(R::sub(fy, T(1)), T(i)), H, align);
        xok[i] = (unsigned)xi < (unsigned)W_;
        yok[i] = (unsigned)yi < (unsigned)H;
        xo[i] = xi;
        yo[i] = yi * W;
      }
      if (PAD == KB200_FILL) {
        T cover = T(0);
#pragma unroll
        for (int i = 0; i < NT; ++i) {
          T r = T(0);
#pragma unroll
          for (int j = 0; j < NT; ++j) r = R::fma((yok[i] && xok[j]) ? T(1) : T(0), cx[j], r);
          cover = R::fma(r, cy[i], cover);
        }
        inv_cover = R::sub(T(1), cover);
      }
    }
  }

  __device__ __forceinline__ T sample(const T* __restrict__ s) const {
    using R = RN<T>;
    if (INTERP == KB200_BILINEAR) {
      T acc = T(0);
      if (ok[0]) acc = R::fma(ldg(s + o), w[0], acc);
      if (ok[1]) acc = R::fma(ldg(s + o + 1), w[1], acc);
      if (ok[2]) acc = R::fma(ldg(s + o + W), w[2], acc);
      if (ok[3]) acc = R::fma(ldg(s + o + W + 1), w[3], acc);
      return acc;
    } else if (INTERP == KB200_NEAREST) {
      return ok[0] ? ldg(s + o) : T(0);
    } else {
      T acc = T(0);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        T r = T(0);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const T v = (yok[i] && xok[j]) ? ldg(s + yo[i] + xo[j]) : T(0);
          r = R::fma(v, cx[j], r);
        }
        acc = R::fma(r, cy[i], acc);
      }
      return acc;
    }
  }

  // The same blend with the taps supplied by ``fetch(offset)`` (offset = row * W + column of the tap, in pixels): lets a
  // kernel whose source is not a planar T image (warp_u8.cuh: interleaved uint8) share the tap order and rounding of
  // sample() without touching it.
  template <typename F>
  __device__ __forceinline__ T sample_with(F fetch) const {
    using R = RN<T>;
    if (INTERP == KB200_BILINEAR) {
      T acc = T(0);
      if (ok[0]) acc = R::fma(fetch(o), w[0], acc);
      if (ok[1]) acc = R::fma(fetch(o + 1), w[1], acc);
      if (ok[2]) acc = R::fma(fetch(o + W), w[2], acc);
      if (ok[3]) acc = R::fma(fetch(o + W + 1), w[3], acc);
      return acc;
    } else if (INTERP == KB200_NEAREST) {
      return ok[0] ? fetch(o) : T(0);
    } else {
      T acc = T(0);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        T r = T(0);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const T v = (yok[i] && xok[j]) ? fetch(yo[i] + xo[j]) : T(0);
          r = R::fma(v, cx[j], r);
        }
        acc = R::fma(r, cy[i], acc);
      }
      return acc;
    }
  }

  // value written for a channel: sample (+ (1 - coverage) * fill for PAD == KB200_FILL)
  __device__ __forceinline__ T finish(T v, T fill) const {
    using R = RN<T>;
    if (PAD == KB200_FILL) return R::add(v, R::mul(inv_cover, fill));
    return v;
  }
};

// Per-sample 3x3 matrix held in registers; the map of A.3 with the reference's association order.
template <typename T>
struct Mat3 {
  T m00, m01, m02, m10, m11, m12, m20, m21, m22;
  __device__ __forceinline__ void load(const T* p) {
    m00 = p[0]; m01 = p[1]; m02 = p[2];
    m10 = p[3]; m11 = p[4]; m12 = p[5];
    m20 = p[6]; m21 = p[7]; m22 = p[8];
  }
};

template <typename T, bool PROJ>
__device__ __forceinline__ void map_point(const Mat3<T>& m, T bx, T by, T& gx, T& gy, T& den) {
  using R = RN<T>;
  // imgwarp.py:167-169 / :279-280: (m_i0 * x + m_i1 * y) + m_i2, then a true division
  T nx = R::add(R::add(R::mul(m.m00, bx), R::mul(m.m01, by)), m.m02);
  T ny = R::add(R::add(R::mul(m.m10, bx), R::mul(m.m11, by)), m.m12);
  if (PROJ) {
    den = R::add(R::add(R::mul(m.m20, bx), R::mul(m.m21, by)), m.m22);
    gx = R::div(nx, den);
    gy = R::div(ny, den);
  } else {
    den = T(1);
    gx = nx;
    gy = ny;
  }
}

}  // namespace kb200
