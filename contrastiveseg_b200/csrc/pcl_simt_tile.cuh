// Tile machinery of the exact fp32 (SIMT) InfoNCE sweep (pcl_infonce_simt.cu: the stock and the top-k modes; pcl_topk.cu
// sizes the top-k scratch by its row tile).
#pragma once
#include "pcl_common.cuh"
#include "pcl_sweep.cuh"

namespace pcl {

constexpr int TM = 64, TN = 64, LDT = 68;     // tile rows/cols, padded leading dim of transposed tiles
constexpr int SWEEP_THREADS = 256;
constexpr int QMAX = 16;                      // D/16 accumulators per row in BWD (D <= 256)

__device__ __forceinline__ const float* col_row(const SweepArgs& a, int64_t n, int& label) {
  if (a.mode == 1) {
    int c = (int)(n / a.R);
    int q = (int)(n - (int64_t)c * a.R);
    label = c + 1;
    return q < a.M0 ? a.segq + ((int64_t)(c + 1) * a.M0 + q) * a.D
                    : a.pixq + ((int64_t)(c + 1) * a.M1 + (q - a.M0)) * a.D;
  }
  if (a.mode == 0) { label = a.acls[n]; return a.anchors + n * a.D; }
  label = a.ccls[n];
  return a.contrast + n * a.D;
}

// Load a 64 x D row-major block (row pointers in s_ptr, nullptr = zero row) transposed into dst[k*LDT + r].
__device__ __forceinline__ void load_tile_T(float* __restrict__ dst, const float* const* s_ptr, int D) {
  const int r = threadIdx.x & 63, kq = threadIdx.x >> 6;
  const float* src = s_ptr[r];
  for (int kk = kq * 8; kk < D; kk += 32) {
    float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
    if (src != nullptr) {
      v0 = *reinterpret_cast<const float4*>(src + kk);
      v1 = *reinterpret_cast<const float4*>(src + kk + 4);
    }
    dst[(kk + 0) * LDT + r] = v0.x; dst[(kk + 1) * LDT + r] = v0.y;
    dst[(kk + 2) * LDT + r] = v0.z; dst[(kk + 3) * LDT + r] = v0.w;
    dst[(kk + 4) * LDT + r] = v1.x; dst[(kk + 5) * LDT + r] = v1.y;
    dst[(kk + 6) * LDT + r] = v1.z; dst[(kk + 7) * LDT + r] = v1.w;
  }
}

// host side (pcl_infonce_simt.cu): descriptor validation + split geometry, shared-memory size of one sweep CTA
// (topk: the four per-row / per-column selection arrays of the top-k modes, 1 KB more)
int simt_make_args(const pcl_sweep_desc* d, SweepArgs* a);
size_t simt_sweep_smem(int D, bool bwd, bool topk);

}  // namespace pcl
