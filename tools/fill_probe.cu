// Zero-fill rate on H100 as a function of the fill's CTA count P (tools/fill_probe.py builds and runs this):
//   excl      1024 threads of 16-byte stores per CTA, every byte of shared memory requested (one CTA owns its SM)
//   bulk      one thread per CTA issues cp.async.bulk stores of a zeroed shared-memory tile over the CTA's contiguous
//             share, `depth` bulk groups in flight; optionally with an L2 evict_first cache policy
// Prints one JSON line per (bytes, variant, P, tile, depth, hint): GB/s over CUDA events around `reps` launches.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

namespace ptx {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// bulk store shared -> global of `bytes` (a multiple of 16, both addresses 16-byte aligned), tracked by bulk groups
__device__ __forceinline__ void bulk_store(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(reinterpret_cast<uint64_t>(gmem_dst)),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// returns once at most N committed groups still read shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// returns once every bulk store of the thread is complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
}  // namespace ptx

__global__ void __launch_bounds__(1024, 1) k_excl(uint4* __restrict__ p, uint64_t n16) {
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) { p[i] = z; p[i + stride] = z; p[i + 2 * stride] = z; p[i + 3 * stride] = z; }
  for (; i < n16; i += stride) p[i] = z;
}

__device__ __forceinline__ void bulk_store_hint(void* dst, const void* src, uint32_t bytes, uint64_t pol) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
               ::"l"(reinterpret_cast<uint64_t>(dst)), "r"(ptx::smem_u32(src)), "r"(bytes), "l"(pol) : "memory");
}

template <int DEPTH, bool HINT>
__global__ void __launch_bounds__(32, 1) k_bulk(uint8_t* __restrict__ p, uint64_t n16, uint32_t tile) {
  extern __shared__ __align__(128) uint8_t s_zero[];
  for (uint32_t i = threadIdx.x; i < tile / 16; i += blockDim.x) reinterpret_cast<uint4*>(s_zero)[i] = make_uint4(0u, 0u, 0u, 0u);
  ptx::fence_proxy_async();
  __syncthreads();
  if (threadIdx.x != 0) return;
  uint64_t pol = 0;
  if (HINT) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  const uint64_t per = n16 / gridDim.x, rem = n16 % gridDim.x;
  const uint64_t b = blockIdx.x * per + min((uint64_t)blockIdx.x, rem), e = b + per + (blockIdx.x < rem ? 1 : 0);
  for (uint64_t o = b * 16; o < e * 16;) {
    const uint32_t n = (uint32_t)min((uint64_t)tile, e * 16 - o);
    if (HINT) bulk_store_hint(p + o, s_zero, n, pol); else ptx::bulk_store(p + o, s_zero, n);
    ptx::bulk_commit();
    ptx::bulk_wait_read<DEPTH - 1>();
    o += n;
  }
  ptx::bulk_wait_all();
}

template <int DEPTH, bool HINT>
static void launch_bulk(int P, uint8_t* p, uint64_t n16, uint32_t tile, size_t smem) {
  k_bulk<DEPTH, HINT><<<P, 32, smem>>>(p, n16, tile);
}

int main(int argc, char** argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 50;
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const uint64_t sizes[2] = {268435456ull, 134217728ull};          // S1 gradient: fp32, and the half-precision gradient
  const int Ps[] = {4, 8, 12, 16, 24, 32, 48, 64, 100};
  uint8_t* buf = nullptr;
  CK(cudaMalloc(&buf, sizes[0]));
  const size_t excl_smem = 232448, bulk_smem = 116 * 1024;
  CK(cudaFuncSetAttribute(k_excl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)excl_smem));
  void (*bulk_fns[4])(int, uint8_t*, uint64_t, uint32_t, size_t) = {launch_bulk<2, false>, launch_bulk<8, false>,
                                                                    launch_bulk<2, true>, launch_bulk<8, true>};
  CK(cudaFuncSetAttribute(k_bulk<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bulk_smem));
  CK(cudaFuncSetAttribute(k_bulk<8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bulk_smem));
  CK(cudaFuncSetAttribute(k_bulk<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bulk_smem));
  CK(cudaFuncSetAttribute(k_bulk<8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bulk_smem));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  auto timed = [&](auto&& launch) {
    for (int i = 0; i < 3; ++i) launch();
    CK(cudaEventRecord(e0));
    for (int i = 0; i < reps; ++i) launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    return ms / reps;
  };
  for (uint64_t bytes : sizes) {
    const uint64_t n16 = bytes / 16;
    for (int P : Ps) {
      if (P > sms) continue;
      const float ms = timed([&] { k_excl<<<P, 1024, excl_smem>>>((uint4*)buf, n16); });
      printf("{\"bytes\": %llu, \"variant\": \"excl\", \"P\": %d, \"us\": %.2f, \"GBps\": %.1f}\n", (unsigned long long)bytes,
             P, ms * 1e3f, bytes / (ms * 1e6f));
      const uint32_t tiles[3] = {16384u, 32768u, 65536u};
      for (int f = 0; f < 4; ++f)
        for (uint32_t tile : tiles) {
          const float mb = timed([&] { bulk_fns[f](P, buf, n16, tile, bulk_smem); });
          printf("{\"bytes\": %llu, \"variant\": \"bulk\", \"P\": %d, \"tile\": %u, \"depth\": %d, \"evict_first\": %d, "
                 "\"us\": %.2f, \"GBps\": %.1f}\n", (unsigned long long)bytes, P, tile, (f & 1) ? 8 : 2, f >> 1,
                 mb * 1e3f, bytes / (mb * 1e6f));
        }
    }
  }
  fflush(stdout);
  CK(cudaFree(buf));
  return 0;
}
