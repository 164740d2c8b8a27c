// What the warp-specialised wgmma kernels share: the tensor-core InfoNCE sweeps (pcl_infonce_tc.cu), the fused
// small-anchor kernel (pcl_infonce_fused.cu) and the projection-head GEMMs (pcl_norm.cu).  Include it after
// ptx_sm90.cuh (the CPU emulator puts a model of that header first on the include path).
#pragma once
#include "pcl_common.cuh"

namespace pcl {

// Tensor map of a bf16 row-major (rows, cols) matrix, cols a multiple of 8: box = 64 columns (128 B) x box_rows,
// 128-byte swizzle, out-of-bounds rows read as zero.  Defined in pcl_infonce_tc.cu.
int tc_make_tmap(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows);

// The dynamic shared memory as a T at its first 1024-byte boundary (the 128-byte swizzle pattern repeats every 1024 B;
// launches request sizeof(T) + 1024).  The offset is added to the array itself, not rounded through an integer: the
// compiler keeps the shared state space and emits LDS / STS instead of generic loads and stores.
template <class T>
__device__ __forceinline__ T& aligned_smem(uint8_t* raw) {
  return *reinterpret_cast<T*>(raw + ((1024u - (ptx::smem_u32(raw) & 1023u)) & 1023u));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Sum of a row over the 4 lanes of a quad (the same fixed order on every lane).
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// CTA layout of the contrast kernels: a 128-row anchor tile against 256-column contrast tiles, D = 256 as 4 K-blocks of
// 64 (128 bytes of bf16 per row: one swizzle row).
namespace cta {
constexpr int BM = 128, BN = 256, BK = 64, NKB = 4, DDIM = 256;
constexpr int A_KB_BYTES = BM * BK * 2;          // 16 KB
constexpr int WG_ROW_BYTES = 64 * 128;           // offset of warpgroup 1's 64 rows inside a [rows x 64] K-block
constexpr int NUM_THREADS = 384;                 // warps 0-7: two consumer warpgroups, warps 8-11: producer warpgroup
constexpr int PRODUCER_WARP = 8;                 // (its first warp issues the TMA loads)
// Registers per thread after setmaxnreg: 2 x 128 x 232 + 128 x 40 fit the 64 K register file; the consumers hold the
// wgmma accumulators (128 floats for an m64n256 tile).
constexpr uint32_t CONSUMER_REGS = 232, PRODUCER_REGS = 40;
constexpr int EPI_THREADS = 256;                 // the consumer warpgroups (named barrier 1; barriers 2, 3: one warpgroup)
constexpr float LN2 = 0.6931471805599453f;
}  // namespace cta

}  // namespace pcl
