// Micro-benchmark: throughput of cp.async.bulk global->shared per SM as a function of the copy size.
// Two CTAs per SM, one issuing warp each, double-buffered: every "tile" is `ncopies` copies of `bytes` bytes whose sources lie
// `pitch` bytes apart (image rows), completion on an mbarrier.  nvcc -arch=sm_90a -O3 -o bulk_rate bulk_rate.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__global__ void __launch_bounds__(32, 2) k(const char* __restrict__ src, size_t src_bytes, int ncopies, int bytes, int pitch, int tiles,
                                            unsigned long long* cycles) {
  extern __shared__ __align__(128) unsigned char sm[];
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(sm);   // 2 barriers
  unsigned char* buf = sm + 128;
  const int lane = threadIdx.x;
  const int buf_bytes = ncopies * bytes;
  if (lane == 0) {
    for (int i = 0; i < 2; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(bar + i)));
    asm volatile("fence.mbarrier_init.release.cluster;");
  }
  __syncwarp();
  const size_t span = (size_t)ncopies * pitch;
  size_t off = ((size_t)blockIdx.x * 7919u * 4096u) % (src_bytes - span - 4096);
  off &= ~(size_t)127;
  const unsigned long long t0 = clock64();
  auto issue = [&](int t) {
    const int b = t & 1;
    if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.release.cta.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar + b)), "r"(buf_bytes) : "memory");
    __syncwarp();
    if (lane < ncopies)
      asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(buf + (size_t)b * buf_bytes + (size_t)lane * bytes)),
                   "l"(src + off + (size_t)lane * pitch), "r"(bytes), "r"(s32(bar + b)) : "memory");
    off += span; if (off + span + 4096 > src_bytes) off = 0;
  };
  issue(0); issue(1);
  for (int t = 0; t < tiles; ++t) {
    const int b = t & 1; const unsigned par = (t >> 1) & 1;
    unsigned ok = 0;
    while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(s32(bar + b)), "r"(par) : "memory");
    if (t + 2 < tiles) issue(t + 2);
  }
  if (lane == 0) atomicMax(cycles, clock64() - t0);
}
int main() {
  const size_t src_bytes = 4ull << 30;
  char* src; cudaMalloc(&src, src_bytes); cudaMemset(src, 1, src_bytes);
  unsigned long long* cyc; cudaMalloc(&cyc, 8);
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  const int grid = p.multiProcessorCount * 2;
  struct Cfg { int n, bytes, pitch; } cfgs[] = {{15, 1088, 5120}, {29, 1088, 5120}, {8, 2176, 5120}, {4, 4352, 5120}, {2, 8192, 8192}, {1, 15360, 15360}, {1, 30720, 30720}, {30, 512, 5120}, {15, 1088, 1088}};
  for (auto c : cfgs) {
    const int tiles = 4000;
    const size_t smem = 128 + 2 * (size_t)c.n * c.bytes;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaMemset(cyc, 0, 8);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k<<<grid, 32, smem>>>(src, src_bytes, c.n, c.bytes, c.pitch, 200, cyc);   // warm
    cudaEventRecord(a);
    k<<<grid, 32, smem>>>(src, src_bytes, c.n, c.bytes, c.pitch, tiles, cyc);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    const double bytes = (double)grid * tiles * c.n * c.bytes;
    printf("copies/tile %2d x %5d B (pitch %5d): %.3f ms  %.1f GB/s total  %.2f GB/s/SM  %.2f Mcopies/s/SM  err=%s\n", c.n, c.bytes, c.pitch, ms,
           bytes / ms / 1e6, bytes / ms / 1e6 / p.multiProcessorCount, (double)grid * tiles * c.n / ms / 1e3 / p.multiProcessorCount, cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}
