// kornia_b200 -- TMA plumbing shared by the tiled kernels: the mbarrier / cp.async.bulk.tensor wrappers (namespace tma),
// the persistent-CTA work split (Segments) and the host side of tensor maps.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>

#include "common.cuh"

namespace kb200 {

namespace tma {
#ifdef KB200_HOST_EMU  // tools/hostemu: the same kernels executed on the CPU, one fiber per thread; never defined under nvcc
#include "../../tools/hostemu/tma_emu.inl"
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 3-D tiled load: box (BW, BH, NC) at element coordinates (c0, c1, c2); completes on `bar`
__device__ __forceinline__ void load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// shared-memory load at a 32-bit shared-space address
// (constant offsets added by the caller are folded into the instruction's immediate by ptxas)
__device__ __forceinline__ float lds(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
// read-only variant (data that no thread writes while it is being read, e.g. the TMA-staged source box): not
// volatile, so the compiler may interleave these loads with the ordered strip updates
__device__ __forceinline__ float lds_ro(uint32_t addr) {
  float v;
  asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v));
}
// true in exactly one lane of a converged warp (the form ptxas needs around uniform-datapath TMA issue)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}
// pull a box into L2 ahead of the real load (no shared memory, no barrier)
__device__ __forceinline__ void prefetch_3d(const CUtensorMap* map, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(map), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void prefetch_map(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// bulk async-group plumbing of the TMA reduce-add (tiled backward kernels)
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void reduce_add_3d(const CUtensorMap* map, uint32_t src_smem, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(src_smem),
               "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void prefetch_l1(size_t global_addr) { asm volatile("prefetch.global.L1 [%0];" ::"l"(global_addr)); }
__device__ __forceinline__ float rcp_approx(float den) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(den));
  return r;
}
#endif  // KB200_HOST_EMU

}  // namespace tma

// Work decomposition shared by the producer and the consumers of a CTA.  A strip is one row of tiles
// of one image.  Full rounds hand whole strips to CTAs round-robin (neighbouring CTAs then work on
// vertically adjacent strips at the same time, so their shared halo rows hit in L2); the strips
// left over after the last full round are cut into equal runs of tiles so every CTA finishes at
// the same time (otherwise the last round leaves most SMs idle: 3 % of the headline launch).
struct Segments {
  int nstrips, tiles_x, rounds, lo, hi;  // leftover tile range [lo, hi) of this CTA
  __device__ Segments(int nstrips_, int tiles_x_) : nstrips(nstrips_), tiles_x(tiles_x_) {
    const int G = gridDim.x, c = blockIdx.x;
    rounds = nstrips / G;
    const long long left = (long long)(nstrips - rounds * G) * tiles_x;
    lo = (int)(left * c / G);
    hi = (int)(left * (c + 1) / G);
  }
  // segment i of this CTA: tiles [tx0, tx1) of `strip`; false when the CTA is done
  __device__ bool get(int i, int& strip, int& tx0, int& tx1, int& cursor) const {
    if (i < rounds) {
      strip = i * gridDim.x + blockIdx.x;
      tx0 = 0;
      tx1 = tiles_x;
      cursor = lo;
      return true;
    }
    if (i == rounds) cursor = lo;
    if (cursor >= hi) return false;
    strip = rounds * gridDim.x + cursor / tiles_x;
    tx0 = cursor - (cursor / tiles_x) * tiles_x;
    tx1 = min(tiles_x, tx0 + (hi - cursor));
    cursor += tx1 - tx0;
    return true;
  }
};

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
    else
      (void)cudaGetLastError();
  }
  return fn;
}

inline int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// fp32 (W, H, planes) tensor map with a (box_w, box_h, box_c) box: rows of W floats, planes of H rows, out-of-image texels
// read as zeros.  false when the driver has no encoder or refuses the map.
inline bool encode_plane_map(CUtensorMap* map, const float* x, long long planes, int H, int W, int box_w, int box_h, int box_c = 1) {
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
  const cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_c};
  const cuuint32_t estr[3] = {1, 1, 1};
  return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace kb200
