// Shared helpers for the pixel-contrast engine kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/pcl.h"

namespace pcl {

// ---- error plumbing -----------------------------------------------------------------------------
void set_cuda_error(cudaError_t e, const char* file, int line);
void set_error_text(const char* text);            // driver-API failures (tensor-map encoding): same per-thread slot

#define PCL_CUDA(expr)                                                  \
  do {                                                                  \
    cudaError_t e__ = (expr);                                           \
    if (e__ != cudaSuccess) {                                           \
      ::pcl::set_cuda_error(e__, __FILE__, __LINE__);                   \
      return PCL_ERR_CUDA;                                              \
    }                                                                   \
  } while (0)

void count_launch();
#define PCL_LAUNCH_CHECK()          \
  do {                              \
    ::pcl::count_launch();          \
    PCL_CUDA(cudaGetLastError());   \
  } while (0)

#define PCL_REQUIRE(cond)                 \
  do {                                    \
    if (!(cond)) return PCL_ERR_ARG;      \
  } while (0)

// ---- input element types (PCL_DT_*) ----------------------------------------------------------------
// Kernels that read the embedding, the logits or the bank keys, and the writers of the dense gradient, are templated
// on the element type.  Loads convert to fp32 (exact); a half gradient is the fp32 value rounded once to nearest-even.
__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }
template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ float from_f32<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float x) { return __float2bfloat16(x); }
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }
static inline bool dtype_ok(int dt) { return dt == PCL_DT_F32 || dt == PCL_DT_BF16 || dt == PCL_DT_F16; }
static inline size_t dtype_size(int dt) { return dt == PCL_DT_F32 ? sizeof(float) : 2; }
// Runs the statements that follow with the type name T bound to the element type of dtype code `dt` (fp32 for 0).
#define PCL_DT_SWITCH(dt, T, ...)                                       \
  switch (dt) {                                                         \
    case PCL_DT_BF16: { using T = __nv_bfloat16; __VA_ARGS__ } break;   \
    case PCL_DT_F16: { using T = __half; __VA_ARGS__ } break;           \
    default: { using T = float; __VA_ARGS__ } break;                    \
  }

// internal (not part of the C ABI): fused variants used by pcl_step_forward / pcl_step_backward.  `embed_dtype` /
// `seg_dtype` / `grad_dtype`: element type of embed and grad_clear / seg / grad_embed (PCL_DT_*).

// Arguments of the selection kernel (pcl_select_gather): the stabiliser and slot initialisation of the tensor path
// (row_m2 .. n_slot_rows), the captured step's counter and timeline (seed_ctr, dbg) and the sparse reset (prev_rows,
// grad_clear) are optional.
struct select_args {
  const pcl_geom* g;
  const void* embed;
  int embed_dtype, normalize;
  uint64_t seed;
  const uint16_t* keys;
  const int32_t *chunk_pref, *plan, *ranks, *prev_rows;
  int32_t* anchor_meta;
  float *anchors_f32, *inv_norm, *norm_max, *row_m2, *partials;
  void *anchors_bf16, *grad_clear;
  float m2_scale;
  int64_t n_slot_rows;
  const unsigned long long* seed_ctr;
  unsigned int* dbg;
};
int select_gather(const select_args& a, void* stream);
int tc_fwd_ex(const pcl_tc_desc* d, float* row_m2, float* partials, float* rowstats, float* loss, void* stream,
              bool skip_prep, unsigned long long* step_counter = nullptr);
int simt_fwd_ex(const pcl_sweep_desc* d, int k, uint32_t* scratch, float* partials, float* rowstats, float* loss,
                void* stream, unsigned long long* step_counter);
int simt_bwd_ex(const pcl_sweep_desc* d, int k, uint32_t* scratch, const float* rowstats, const float* grad_loss,
                float* dpartials, float* dA, void* stream);
int tc_fwd_topk_ex(const pcl_tc_desc* d, int k, uint32_t* scratch, float* row_m2, float* partials, float* rowstats,
                   float* loss, void* stream, bool skip_prep, unsigned long long* step_counter);
int tc_query(const pcl_tc_desc* d, int64_t* n_slot_rows, float* m2_scale);
int tc_bwd_ex(const pcl_tc_desc* d, const float* row_m2, const float* rowstats, const float* grad_loss, float* dpartials,
              float* dA, void* stream, int* splits_out, int* a_pad_out, const uint32_t* topk_scratch = nullptr);

int self_fused_supported(const pcl_tc_desc* d);
// layout of the fused kernel's partial gradient rows, dpartials [splits][a_pad][256]: split p holds the contrast
// columns [p * split_cols, (p + 1) * split_cols)
void self_fused_splits(int a_rows, int* a_pad, int* splits, int* split_cols);
int self_fused(const pcl_tc_desc* d, const float* row_m2, float* partials, float* rowstats, float* loss, float* dpartials,
               unsigned int* sync, void* stream);
int class_stats(const pcl_geom* g, const int64_t* labels, const void* seg, const int64_t* predict, uint16_t* keys,
                int32_t* chunk_pref, int32_t* counts, int32_t* plan, unsigned int* done_ctr, void* stream, int seg_dtype);
int fill_zero(void* ptr, uint64_t bytes, void* stream, unsigned int* dbg, int reserve_sms);

// Where the dense gradient's anchor rows come from: the (A, D) matrix dA (with the projection of the L2 normalise when
// `normalize`: anchors_f32, inv_norm), or, when dpartials is set, the backward sweep's per-split partial rows (dpartials
// [splits][a_pad][D]; split_cols > 0: split p covers the contrast columns [p * split_cols, (p + 1) * split_cols) and only
// the live ones were written), summed in fixed order and scaled by inv_T * grad_scale[0].
struct grad_rows {
  const float *dA, *anchors_f32, *inv_norm, *dpartials, *grad_scale;
  int normalize, splits, split_cols, a_pad;
  float inv_T;
};
// Writes the dense (B, D, h, w) gradient; `zeroed`: the caller has zero-filled it already.  The captured fused step's
// extras (dbg: its timeline, step_counter, prev_rows: what the next step's sparse reset clears) serve partial rows into a
// zeroed buffer.
int dense_grad(const pcl_geom* g, const int32_t* plan, const int32_t* anchor_meta, const grad_rows& r, bool zeroed,
               void* grad_embed, int grad_dtype, void* stream, unsigned int* dbg = nullptr,
               unsigned long long* step_counter = nullptr, int32_t* prev_rows = nullptr);

// ---- per-device kernel attributes ----------------------------------------------------------------
// cudaFuncAttributeMaxDynamicSharedMemorySize is a property of (function, device) and SETS the limit (a later call with
// a smaller size lowers it).  Every kernel therefore opts in ONCE per device to the largest size it can ever need
// (known at compile time: D <= 256); the bit mask is indexed by the current device, so a process that drives several
// GPUs gets every device configured.
struct SmemOptIn { unsigned long long mask; };
template <typename F>
static inline int smem_opt_in(SmemOptIn& st, F func, size_t max_bytes) {
  int dev = 0;
  PCL_CUDA(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (__atomic_load_n(&st.mask, __ATOMIC_ACQUIRE) & bit) return PCL_OK;
  PCL_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_bytes));
  __atomic_fetch_or(&st.mask, bit, __ATOMIC_RELEASE);
  return PCL_OK;
}
#define PCL_SMEM_OPT_IN(func, max_bytes)                                   \
  do {                                                                      \
    static ::pcl::SmemOptIn st__ = {0ull};                                  \
    int rc__ = ::pcl::smem_opt_in(st__, func, (max_bytes));                 \
    if (rc__ != PCL_OK) return rc__;                                        \
  } while (0)

// SM count of the current device (cached per device; 132 when sizing on a host without one)
int num_sms();

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---- optional in-graph timeline (diagnostics) ----------------------------------------------------------
// The step's `sync` buffer (pcl_step_desc.sync, >= 1024 words) doubles as a timeline when word 7 is non-zero: words
// [16, 16 + 4*16) hold, per kernel slot k, {min block start, max block end} of %globaltimer (ns) — the only way to see
// how the kernels of a captured graph actually overlap (ncu serialises them).  Costs one predicated load per block when off.
enum { PCL_TL_KEYS = 0, PCL_TL_SELECT = 1, PCL_TL_FUSED = 2, PCL_TL_SCATTER = 3, PCL_TL_FILL = 4 };
__device__ __forceinline__ unsigned long long pcl_globaltimer() {
#ifdef PCL_EMULATION
  return 0ull;
#else
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
#endif
}
__device__ __forceinline__ void tl_begin(unsigned int* dbg, int slot) {
  if (dbg != nullptr && dbg[7] != 0u && threadIdx.x == 0)
    atomicMin(reinterpret_cast<unsigned long long*>(dbg + 16) + 2 * slot, pcl_globaltimer());
}
__device__ __forceinline__ void tl_end(unsigned int* dbg, int slot) {
  if (dbg != nullptr && dbg[7] != 0u && threadIdx.x == 0)
    atomicMax(reinterpret_cast<unsigned long long*>(dbg + 16) + 2 * slot + 1, pcl_globaltimer());
}

// ---- device helpers -------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// wgmma accumulator fragment -> row view.  The tensor-core epilogues work on one row per thread and 32 consecutive
// columns at a time, while the accumulator of an m64nN wgmma is spread over the warpgroup (layout: ptx_sm90.cuh).
// frag_store_cols writes columns [8 i0, 8 (i0 + NI)) of warpgroup thread t's fragment to dst[row * pitch + column - 8 i0];
// after a barrier of the warpgroup, load_row32 reads 32 consecutive columns of one row back.  A pitch of 4 (mod 32)
// floats keeps the 16-byte row reads free of bank conflicts.
template <int NI, int NF>
__device__ __forceinline__ void frag_store_cols(const float (&d)[NF], int i0, float* dst, int pitch, int t) {
  const int row = 16 * (t >> 5) + ((t & 31) >> 2), col = 2 * (t & 3);
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(dst + (row + 8 * h) * pitch + 8 * i + col) =
          make_float2(d[4 * (i0 + i) + 2 * h], d[4 * (i0 + i) + 2 * h + 1]);
}
__device__ __forceinline__ void load_row32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 x = reinterpret_cast<const float4*>(src)[q];
    v[4 * q] = __float_as_uint(x.x); v[4 * q + 1] = __float_as_uint(x.y);
    v[4 * q + 2] = __float_as_uint(x.z); v[4 * q + 3] = __float_as_uint(x.w);
  }
}

// Class rank used for the sorted anchor layout: 1,2,...,K-1,0  (class 0 last: in bank mode its
// positives are the analytic zero tail, Q3).
__device__ __host__ __forceinline__ int class_rank(int c, int K) { return c == 0 ? K - 1 : c - 1; }

// ATen nearest-neighbour source index (UpSampleNearest: min(int(floorf(dst*scale)), in-1), scale=in/out in fp32).
__device__ __host__ __forceinline__ int nearest_src(int dst, float scale, int in_size) {
  int s = (int)floorf((float)dst * scale);
  return s < in_size - 1 ? s : in_size - 1;
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Keyed bijection on [0, n): an 8-round balanced Feistel network on the next even number of bits, with cycle walking.
// Used when no permutation table is injected: view j of a group takes element perm(j), so distinct j give distinct
// elements without any sequential state (replaces torch.randperm(n)[:k]).  The round function hashes (key, round, half)
// with the full 64-bit key, so small groups are sampled without the pairwise structure of multiply/xorshift rounds
// (measured on n = 60, k = 10: pair co-occurrence chi2/dof ~1.0, was 3.1; n = 7, k = 3: ~1.0, was 26;
// tests/test_host_logic.py checks the host model of this function, tests/test_emu_kernels.py that the kernels follow it).
__device__ __forceinline__ uint32_t keyed_perm(uint32_t j, uint32_t n, uint64_t key) {
  if (n <= 1) return 0;
  const int bits = 32 - __clz(n - 1);                  // ceil(log2 n) >= 1
  const int hb = (bits + 1) >> 1;                      // half width (<= 16): the network permutes [0, 2^(2 hb)) >= [0, n)
  const uint32_t hmask = (1u << hb) - 1u;
  uint32_t x = j;
  do {
    uint32_t L = x >> hb, R = x & hmask;
#pragma unroll
    for (int r = 0; r < 8; ++r) {                       // 4 rounds leave visible structure on domains of 16 elements
      const uint32_t f = (uint32_t)mix64(key + (uint64_t)r * 0x9E3779B97F4A7C15ull + R) & hmask;
      const uint32_t t = R;
      R = L ^ f;
      L = t;
    }
    x = (L << hb) | R;
  } while (x >= n);                                    // domain <= 4n: a few iterations at most on average
  return x;
}

}  // namespace pcl
