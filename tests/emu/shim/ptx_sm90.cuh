// TEST INFRASTRUCTURE — functional model of the sm_90a primitives behind contrastiveseg_b200/csrc/ptx_sm90.cuh (same
// names and signatures), so that the tensor-path kernels (pcl_infonce_tc.cu, pcl_infonce_fused.cu) run on the
// host-fiber emulator:
//   mbarrier      phase bit + pending arrivals + pending transaction bytes, polled cooperatively
//   TMA           2-D bf16 box copy global -> shared with the SWIZZLE_128B pattern (16-byte chunk index XOR row % 8),
//                 out-of-range rows zero-filled, completes its bytes on the mbarrier later (asynchronous engine)
//   wgmma         m64nNk16 bf16 -> fp32: every thread of the warpgroup computes its own accumulator fragment elements
//                 (layout of the product header), operands fetched through the shared-memory matrix descriptors
//                 (K-major / MN-major, 128-byte swizzle, LBO / SBO) exactly as the real header encodes them
// The wgmma model executes at issue, so it checks indexing, fragment layout, descriptors and the barrier protocol
// (phases, counts, deadlocks) — not the hardware's asynchrony or memory ordering.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace ptx {

constexpr uint32_t SMEM_HANDLE_BASE = 0x400;        // shared-window address of the first byte of dynamic shared memory

inline uint32_t smem_u32(const void* p) {
  const uintptr_t base = (uintptr_t)emu::g_blk->dyn, q = (uintptr_t)p;
  if (q < base || q >= base + emu::g_blk->dyn_bytes) { fprintf(stderr, "emu: smem_u32 of a pointer outside dynamic shared memory\n"); abort(); }
  return (uint32_t)(q - base) + SMEM_HANDLE_BASE;
}
inline uint8_t* smem_ptr(uint32_t handle) { return (uint8_t*)emu::g_blk->dyn + (handle - SMEM_HANDLE_BASE); }

// ---- mbarrier: [0,20) pending arrivals | [20,40) arrival count per phase | [40,63) pending tx bytes | 63 phase ----
struct MbarView {
  uint64_t* w;
  uint64_t pending() const { return *w & 0xFFFFF; }
  uint64_t count() const { return (*w >> 20) & 0xFFFFF; }
  int64_t tx() const { return (int64_t)((*w >> 40) & 0x7FFFFF); }
  uint64_t phase() const { return *w >> 63; }
  void set(uint64_t pend, uint64_t cnt, int64_t tx_, uint64_t ph) { *w = (pend & 0xFFFFF) | ((cnt & 0xFFFFF) << 20) | (((uint64_t)tx_ & 0x7FFFFF) << 40) | (ph << 63); }
  void settle() { if (pending() == 0 && tx() == 0) set(count(), count(), 0, phase() ^ 1); }
};
inline void mbar_init(uint64_t* bar, uint32_t count) { MbarView{bar}.set(count, count, 0, 0); }
inline void fence_barrier_init() {}
inline void fence_proxy_async() {}
inline void mbar_arrive(uint64_t* bar) {
  MbarView b{bar};
  if (b.pending() == 0) { fprintf(stderr, "emu: mbarrier over-arrival\n"); abort(); }
  b.set(b.pending() - 1, b.count(), b.tx(), b.phase());
  b.settle();
}
inline void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  MbarView b{bar};
  if (b.pending() == 0) { fprintf(stderr, "emu: mbarrier over-arrival\n"); abort(); }
  b.set(b.pending() - 1, b.count(), b.tx() + bytes, b.phase());
  b.settle();
}
inline void mbar_complete_tx(uint64_t* bar, uint32_t bytes) {
  MbarView b{bar};
  b.set(b.pending(), b.count(), b.tx() - (int64_t)bytes, b.phase());
  b.settle();
}
// a failed poll hands the processor to the other fibers of the block (every polling loop in the kernels goes through here)
inline bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  const bool ok = MbarView{bar}.phase() != (uint64_t)(parity & 1u);
  if (!ok) emu::spin_yield();
  return ok;
}
inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 16)) {
      fprintf(stderr, "emu: mbarrier timeout block (%u,%u) thread %u parity %u\n", blockIdx.x, blockIdx.y, threadIdx.x, parity);
      abort();
    }
  }
}
inline void bar_sync(int id, int n) { emu::named_barrier(id, n); }
template <uint32_t N> inline void setmaxnreg_dec() {}
template <uint32_t N> inline void setmaxnreg_inc() {}

// ---- TMA ----
struct TmapModel { const uint8_t* base; uint64_t rows; uint64_t row_bytes; uint32_t box_cols; uint32_t box_rows; uint32_t magic; };
inline void prefetch_tmap(const CUtensorMap*) {}
inline bool async_eager() { static const bool e = [] { const char* v = getenv("PCL_EMU_ASYNC"); return v && v[0] == 'e'; }(); return e; }
template <class F> inline void issue_async(int engine, F&& op) {
  if (async_eager()) op();                                   // PCL_EMU_ASYNC=eager: complete at issue time
  else emu::g_blk->async_q.push_back(emu::Block::AsyncOp{engine, std::function<void()>(std::forward<F>(op))});
}
inline void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1) {
  const TmapModel t = *reinterpret_cast<const TmapModel*>(m);
  if (t.magic != 0x7A3Du || t.box_cols * 2 != 128) { fprintf(stderr, "emu: bad tensor map\n"); abort(); }
  if (((uintptr_t)smem_dst & 1023) != 0) { fprintf(stderr, "emu: TMA destination not 1024-byte aligned\n"); abort(); }
  uint8_t* dst = (uint8_t*)smem_dst;
  issue_async(0, [=]() {
    for (uint32_t r = 0; r < t.box_rows; ++r) {
      const int64_t row = (int64_t)c1 + r;
      for (uint32_t c = 0; c < 8; ++c) {
        uint8_t* d = dst + (size_t)r * 128 + ((c ^ (r & 7u)) * 16);
        if (row >= 0 && (uint64_t)row < t.rows) memcpy(d, t.base + (size_t)row * t.row_bytes + ((size_t)c0 + c * 8) * 2, 16);
        else memset(d, 0, 16);
      }
    }
    mbar_complete_tx(bar, t.box_rows * 128);
  });
}

// ---- wgmma ----
inline void wgmma_fence() {}
inline void wgmma_commit() {}
template <int N> inline void wgmma_wait() {}
template <int NF> inline void fence_operands(float (&)[NF]) {}
inline float operand(uint64_t desc, bool mn_major, uint32_t idx, uint32_t k) {
  const uint32_t base = (uint32_t)(desc & 0x3FFF) << 4;
  const uint32_t lbo = (uint32_t)((desc >> 16) & 0x3FFF) << 4, sbo = (uint32_t)((desc >> 32) & 0x3FFF) << 4;
  if (((desc >> 62) & 3) != 1 || ((desc >> 49) & 7) != 0) { fprintf(stderr, "emu: only SWIZZLE_128B descriptors are modelled\n"); abort(); }
  uint32_t L = mn_major ? base + (idx / 64) * lbo + (k / 8) * sbo + (k % 8) * 128 + (idx % 64) * 2
                        : base + (idx / 8) * sbo + (idx % 8) * 128 + k * 2;
  const uint32_t P = L ^ (((L >> 7) & 7u) << 4);
  __nv_bfloat16 h;
  memcpy(&h, smem_ptr(P), 2);
  return __bfloat162float(h);
}
// d (+)= A . B^T for the fragment elements of this thread (A: 64 x 16 K-major; B: N x 16, K-major or MN-major)
template <int TRANS_B, int NF>
inline void wgmma_model(float (&d)[NF], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  const uint32_t t = threadIdx.x & 127u;
  for (int j = 0; j < NF; ++j) {
    const uint32_t i = j / 4, h = (j / 2) & 1, e = j & 1;
    const uint32_t row = 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h, col = 8 * i + 2 * (t & 3) + e;
    float acc = accumulate ? d[j] : 0.f;
    for (uint32_t k = 0; k < 16; ++k) acc += operand(desc_a, false, row, k) * operand(desc_b, TRANS_B != 0, col, k);
    d[j] = acc;
  }
}
template <int TRANS_B>
inline void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  wgmma_model<TRANS_B>(d, desc_a, desc_b, accumulate);
}
template <int TRANS_B>
inline void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  wgmma_model<TRANS_B>(d, desc_a, desc_b, accumulate);
}

// ---- descriptors: identical to the product header (the kernels build them, the model above decodes them) ----
inline uint64_t make_desc_kmajor_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
inline uint64_t make_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

inline float ex2_approx(float x) { return exp2f(x); }
inline float lg2_approx(float x) { return log2f(x); }
inline float rcp_approx(float x) { return 1.f / x; }

}  // namespace ptx
