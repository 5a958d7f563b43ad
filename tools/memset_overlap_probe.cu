// Probe: does cudaMemsetAsync on a second stream make progress while a kernel owns every thread slot of every SM, and
// can that kernel see a cuStreamWriteValue32 that follows the memset?  Decides whether the zero-fill of d/dsrc (0.19 ms of the
// 2.33 ms cfg4 step) can be taken off the critical path with chunked memsets + flags polled by the backward kernel.
// Every wait in the kernels is bounded by %globaltimer: nothing here can hang the device.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/memset_overlap_probe tools/memset_overlap_probe.cu
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);      \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)

__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Fills every thread slot (2 x 1024 threads per SM) and spins for `ns`.
__global__ void __launch_bounds__(1024, 2) spin_kernel(unsigned long long ns, unsigned long long* t_start, unsigned long long* t_end) {
  const unsigned long long t0 = now_ns();
  if (blockIdx.x == 0 && threadIdx.x == 0) *t_start = t0;
  while (now_ns() - t0 < ns) {
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *t_end = now_ns();
}

// Same, but every CTA polls flags[0..nflags) in order and records when block 0 saw each; gives up after `ns`.
__global__ void __launch_bounds__(1024, 2) poll_kernel(unsigned long long ns, const volatile unsigned* flags, int nflags, unsigned long long* seen,
                                                       const float* buf, size_t chunk_floats, int* nonzero) {
  const unsigned long long t0 = now_ns();
  if (blockIdx.x == 0 && threadIdx.x == 0) seen[nflags] = t0;
  for (int i = 0; i < nflags; ++i) {
    while (flags[i] == 0u && now_ns() - t0 < ns) {
    }
    __threadfence();
    if (blockIdx.x == 0 && threadIdx.x == 0) seen[i] = flags[i] ? now_ns() : 0ull;
    // the chunk behind flag i must read as zeros now (sample a few words spread over the chunk)
    if (flags[i]) {
      const size_t at = (size_t)i * chunk_floats + ((size_t)blockIdx.x * 1024 + threadIdx.x) * 997 % chunk_floats;
      if (__ldcg(buf + at) != 0.f) atomicAdd(nonzero, 1);
    }
  }
}

__global__ void fill_kernel(float4* p, size_t n, float v) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = make_float4(v, v, v, v);
}

int main() {
  CK(cudaSetDevice(0));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  const size_t bytes = 128ull * 3 * 720 * 1280 * 4;  // d/dsrc of cfg4: 1.4 GB
  float* buf;
  CK(cudaMalloc(&buf, bytes));
  cudaStream_t a, b;
  CK(cudaStreamCreateWithFlags(&a, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&b, cudaStreamNonBlocking));
  cudaEvent_t e0, e1, k0, k1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&k0)); CK(cudaEventCreate(&k1));
  unsigned long long* stamps;
  CK(cudaMalloc(&stamps, 64 * sizeof(unsigned long long)));
  float ms;

  // 1. memset and a fill kernel alone
  for (int rep = 0; rep < 3; ++rep) {
    CK(cudaEventRecord(e0, b));
    CK(cudaMemsetAsync(buf, 0, bytes, b));
    CK(cudaEventRecord(e1, b));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("memset alone            : %.3f ms  %.0f GB/s\n", ms, bytes / ms * 1e-6);
  }
  for (int rep = 0; rep < 3; ++rep) {
    CK(cudaEventRecord(e0, b));
    fill_kernel<<<sms * 8, 256, 0, b>>>(reinterpret_cast<float4*>(buf), bytes / 16, 0.f);
    CK(cudaEventRecord(e1, b));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("fill kernel alone       : %.3f ms  %.0f GB/s\n", ms, bytes / ms * 1e-6);
  }

  // 2. memset while a kernel owns every thread slot for 4 ms
  for (int rep = 0; rep < 3; ++rep) {
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(k0, a));
    spin_kernel<<<sms * 2, 1024, 0, a>>>(4000000ull, stamps, stamps + 1);
    CK(cudaEventRecord(k1, a));
    CK(cudaEventRecord(e0, b));
    CK(cudaMemsetAsync(buf, 0, bytes, b));
    CK(cudaEventRecord(e1, b));
    CK(cudaDeviceSynchronize());
    float t_mem, t_kern, mem_end_after_kernel_start;
    CK(cudaEventElapsedTime(&t_mem, e0, e1));
    CK(cudaEventElapsedTime(&t_kern, k0, k1));
    CK(cudaEventElapsedTime(&mem_end_after_kernel_start, k0, e1));
    printf("memset under a full grid: memset %.3f ms, kernel %.3f ms, memset done %.3f ms after the kernel began -> %s\n", t_mem, t_kern,
           mem_end_after_kernel_start, mem_end_after_kernel_start < t_kern - 0.5f ? "OVERLAPS (not an SM kernel, or co-resident)" : "SERIALISED");
  }

  // 3. chunked memsets + cuStreamWriteValue32 flags polled by the resident kernel
  typedef CUresult (*WriteValueFn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
  WriteValueFn write_value = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CK(cudaGetDriverEntryPoint("cuStreamWriteValue32", reinterpret_cast<void**>(&write_value), cudaEnableDefault, &qres));
  if (!write_value || qres != cudaDriverEntryPointSuccess) {
    printf("cuStreamWriteValue32 unavailable\n");
    return 0;
  }
  const int nchunks = 8;
  unsigned* flags;
  int* nonzero;
  CK(cudaMalloc(&flags, 64 * sizeof(unsigned)));
  CK(cudaMalloc(&nonzero, sizeof(int)));
  const size_t chunk = bytes / nchunks;
  for (int rep = 0; rep < 3; ++rep) {
    fill_kernel<<<sms * 8, 256, 0, a>>>(reinterpret_cast<float4*>(buf), bytes / 16, 1.f);  // dirty the buffer
    CK(cudaMemsetAsync(flags, 0, 64 * sizeof(unsigned), a));
    CK(cudaMemsetAsync(nonzero, 0, sizeof(int), a));
    CK(cudaMemsetAsync(stamps, 0, 64 * sizeof(unsigned long long), a));
    CK(cudaEventRecord(k0, a));
    CK(cudaStreamWaitEvent(b, k0, 0));
    poll_kernel<<<sms * 2, 1024, 0, a>>>(20000000ull, flags, nchunks, stamps, buf, chunk / 4, nonzero);  // resident before the memsets are enqueued
    CK(cudaEventRecord(k1, a));
    for (int i = 0; i < nchunks; ++i) {
      CK(cudaMemsetAsync(reinterpret_cast<char*>(buf) + i * chunk, 0, chunk, b));
      CUresult r = write_value(b, (CUdeviceptr)(flags + i), 1u, 0);
      if (r != CUDA_SUCCESS) {
        printf("cuStreamWriteValue32 failed: %d\n", (int)r);
        return 0;
      }
    }
    CK(cudaEventRecord(e1, b));
    CK(cudaDeviceSynchronize());
    unsigned long long h[64];
    int bad;
    CK(cudaMemcpy(h, stamps, sizeof(h), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&bad, nonzero, sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaEventElapsedTime(&ms, k0, k1));
    printf("flags seen by the resident kernel (us after its start):");
    for (int i = 0; i < nchunks; ++i) printf(" %s%.0f", h[i] ? "" : "NEVER ", h[i] ? (h[i] - h[nchunks]) * 1e-3 : 0.0);
    printf("; kernel span %.3f ms; non-zero samples behind a raised flag: %d\n", ms, bad);
  }
  return 0;
}
