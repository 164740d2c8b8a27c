// Tensor-core InfoNCE sweep for sm_90a (SURVEY §8 row a6: "anchor x memory-bank similarity as a dense bf16
// contraction on the tensor cores fed by TMA staging").
//
// One CTA = one 128-row anchor tile x a contiguous range of 256-column contrast tiles, D = 256 (K-major bf16):
//   warp 8       TMA producer : anchor tile once (4 x [128 x 64] boxes, 64 KB), then a 3-stage ring of [256 x 64]
//                               contrast boxes (32 KB each), SWIZZLE_128B
//   warps 0-7    two consumer warpgroups, 64 anchor rows each: wgmma m64n256k16 (16 per logit tile, fp32 accumulators
//                in registers), then the epilogue on the same threads: the accumulator goes through a shared-memory
//                staging buffer 32 columns at a time (one row per thread), one FFMA + one ex2 per logit (scale 1/T and
//                the row stabiliser folded into the FFMA), class test only on tiles that straddle a class boundary,
//                row sums kept in registers; never materialises A x N
// Sweeps: NEG (sum over negatives of exp(l - m)), POS (log-prob sums over the positive column range).  The row
// stabiliser is the Cauchy-Schwarz bound m_i = |a_i| * max|c| / T (exact in real arithmetic; no running max needed).
// Partials per (split, row) are combined in fixed order by the shared row-statistic kernels (pcl_sweep.cuh).
#include "pcl_common.cuh"
#include "pcl_sweep.cuh"
#include "ptx_sm90.cuh"
#include "pcl_wgmma.cuh"
#include "pcl_topk.cuh"
#include <mutex>

namespace pcl {
namespace tc {
using namespace cta;

// Forward tile = 128 rows x 256 columns: each consumer warpgroup runs M64 x N256 x K16 wgmmas on its 64 rows, so both
// read the same contrast box once per K step (the widest N wgmma has, the fewest operand bytes per MMA).
constexpr int STAGES = 3;
constexpr int B_STAGE_BYTES = BN * BK * 2;       // 32 KB
constexpr int CONSUMER_WARPS = 8;                // arrivals on an "empty" barrier: every consumer warp after its wgmma wait
constexpr int SPITCH = 36;                       // staging row pitch in floats (32 columns + 4: conflict-free row reads)
constexpr float LOG2E = 1.4426950408889634f;

struct TcArgs {
  const int32_t* acls; const int32_t* diag; const int32_t* plan; const int32_t* ccls;
  const float* row_m2;         // per-row stabiliser in log2 units
  const int32_t* cls_start;    // mode 2 + sorted: first column of every label (PCL_MAX_CLASSES + 1 entries)
  int a_rows, a_pad, mode, K, R, sorted;
  int64_t n_cols;
  float k1;                    // log2(e) / T
  int splits;                  // 2-D grid: column splits per row tile
  int slots;                   // partial slots per row (stride of the partial arrays)
  int tail_count;              // analytic all-zero columns of label 0 (bank mode: R)
  int neg_grid;                // CTAs of the persistent NEG sweep (bounds the partial slots a row tile can own)
  int persistent;              // 1: grid = CTAs, each walks a contiguous range of (row tile, column tile) pairs
  uint32_t r_mul, r_sh;        // exact n / R for 32-bit n without a hardware divide: ((umulhi(n, r_mul) + n') >> r_sh), see div_R
  // a10 (top-k hard negatives on the tensor path): per-row radix bins [a_pad][2048] and the selection state [4][a_rows]
  // (pcl_topk.cuh); NULL = all negatives (the reference).  The selection key is the float x = rn(s * k1) (log2 units),
  // formed with the same instruction in every sweep and in the backward.
  uint32_t* tk_hist;
  const uint32_t* tk_sel;
};

// n / R by multiplication (Granlund-Montgomery round-up method, exact for every 32-bit n): the bank-mode column label
// n / R + 1 is evaluated per 32-column chunk by every epilogue thread, and the integer divide is about 25 instructions.
__device__ __forceinline__ uint32_t div_R(const TcArgs& a, uint32_t n) {
  const uint32_t t = __umulhi(n, a.r_mul);
  return (t + ((n - t) >> 1)) >> a.r_sh;
}
static inline void make_div(uint32_t d, uint32_t* mul, uint32_t* sh) {
  // d >= 1.  l = ceil(log2 d); m = floor(2^32 (2^l - d) / d) + 1; q = (t + ((n - t) >> 1)) >> (l - 1), t = umulhi(m, n)
  uint32_t l = 0;
  while ((1ull << l) < d) ++l;
  if (l == 0) { *mul = 0u; *sh = 0u; return; }                  // d == 1: t = 0 -> (n >> 1) >> ... handled below
  const unsigned long long m = ((1ull << 32) * ((1ull << l) - d)) / d + 1ull;
  *mul = (uint32_t)m;
  *sh = l - 1;
}

struct SmemLayout {
  uint8_t a[NKB * A_KB_BYTES];
  uint8_t c[STAGES * B_STAGE_BYTES];
  float stage[2][2][64][SPITCH];                 // [warpgroup][column half][row]: one 32-column chunk of each half
  uint64_t full[STAGES], empty[STAGES], a_full, a_empty;
  float comb[3][2][BM];
};
static_assert(sizeof(SmemLayout) + 1024 <= 227 * 1024, "shared memory of one H100 block");

// The contrast ring, as the consumer warpgroups walk it: wait for a stage, issue its wgmmas, and release the stage
// before once its wgmmas have retired (one wgmma group stays in flight behind the issue).
struct Ring {
  uint32_t stage = 0, phase = 0;
  int prev = -1;
  __device__ __forceinline__ void release_prev(uint64_t* empty, int lane) {
    if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
    prev = -1;
  }
};

// acc = X . Y^T over D = 256 (4 K-blocks), both K-major: the operand that stays (`fixed`, one [rows x 64] box per
// K-block at `fixed_kb_bytes`) and the one streamed through the ring (one K-block per stage).  RING_IS_A: the ring feeds
// the M side (the transposed POS sweep), else the N side.
template <int STAGES_, int RING_BYTES, bool RING_IS_A, int NF>
__device__ __forceinline__ void ring_mma(float (&acc)[NF], uint32_t fixed_base, uint32_t fixed_kb_bytes, uint32_t ring_base,
                                         uint64_t* full, uint64_t* empty, Ring& ring, int lane) {
  ptx::wgmma_fence();
#pragma unroll 1
  for (int kb = 0; kb < NKB; ++kb) {
    ptx::mbar_wait(&full[ring.stage], ring.phase);
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t df = ptx::make_desc_kmajor_sw128(fixed_base + kb * fixed_kb_bytes + k * 32);
      const uint64_t dr = ptx::make_desc_kmajor_sw128(ring_base + ring.stage * RING_BYTES + k * 32);
      const uint64_t da = RING_IS_A ? dr : df, db = RING_IS_A ? df : dr;
      if constexpr (NF == 128) ptx::wgmma_m64n256k16<0>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
      else ptx::wgmma_m64n64k16<0>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
    }
    ptx::wgmma_commit();
    if (kb > 0) {
      ptx::wgmma_wait<1>();
      ring.release_prev(empty, lane);
    }
    ring.prev = (int)ring.stage;
    if (++ring.stage == STAGES_) { ring.stage = 0; ring.phase ^= 1; }
  }
  ptx::wgmma_wait<0>();
  ring.release_prev(empty, lane);
  ptx::fence_operands(acc);
}

__device__ __forceinline__ int col_label(const TcArgs& a, int n) {      // columns < 2^31
  return a.ccls ? a.ccls[n] : (a.mode == 1 ? (int)div_R(a, (uint32_t)n) + 1 : a.acls[n]);
}

// First / last label of N consecutive 32-column chunks starting at column `base` (lo = -2 / hi = -3: chunk not complete
// or test disabled).  Bank mode with class blocks of R >= 32 N rows: the N chunks meet at most ONE class boundary, so one
// n / R for `base` and comparisons against the next block start replace 2 N multiply-shift divisions.  (Fewer
// instructions; they are evaluated one tile ahead, inside the wait for the accumulator.)
template <int N>
__device__ __forceinline__ void chunk_labels(const TcArgs& a, int base, bool en, int64_t ncols, int (&lo)[N], int (&hi)[N]) {
  if (a.ccls == nullptr && a.mode == 1 && a.R >= 32 * N) {
    const int q = (int)div_R(a, (uint32_t)base);
    const long long nb = (long long)(q + 1) * a.R;                 // first column of the next class block
#pragma unroll
    for (int ch = 0; ch < N; ++ch) {
      const int cb = base + ch * 32;
      const bool in = en && cb + 32 <= ncols;
      lo[ch] = in ? q + 1 + (cb >= nb ? 1 : 0) : -2;
      hi[ch] = in ? q + 1 + (cb + 31 >= nb ? 1 : 0) : -3;
    }
  } else {
#pragma unroll
    for (int ch = 0; ch < N; ++ch) {
      const int cb = base + ch * 32;
      const bool in = en && cb + 32 <= ncols;
      lo[ch] = in ? col_label(a, cb) : -2;
      hi[ch] = in ? col_label(a, cb + 31) : -3;
    }
  }
}

enum { TC_NEG = 0, TC_POS = 1, TC_DUMP = 2,     // DUMP: raw logit tiles to global (descriptor self-test)
       TC_H1 = 3, TC_H2 = 4, TC_H3 = 5,         // a10: radix-select histogram sweeps (11 + 11 + 10 bits of the logit key)
       TC_NEGW = 6 };                           // a10: negative sum with the selection weights

// A segment = consecutive column tiles [ct0, ct1) of one row tile, whose partial row sums go to slot `slot`.
struct Seg { int r, ct0, ct1, slot; };

// Every role (TMA / MMA / epilogue) walks the same deterministic list of segments.
struct SegWalker {
  long long p, p_end, P;
  int T, G, k;
  bool persistent, pending;
  Seg single;
  __device__ __forceinline__ bool next(Seg& s) {
    if (!persistent) {
      if (!pending) return false;
      pending = false;
      s = single;
      return true;
    }
    if (p >= p_end) return false;
    const int r = (int)(p / T);
    const int ct0 = (int)(p - (long long)r * T);
    const long long take = min((long long)(T - ct0), p_end - p);
    // ordinal of this CTA among the CTAs that touch row tile r (CTA j owns pairs [j*P/G, (j+1)*P/G))
    const long long rT = (long long)r * T;
    long long kf = (rT * G) / P;
    while (((kf + 1) * P) / G <= rT) ++kf;
    while (kf > 0 && (kf * P) / G > rT) --kf;
    s.r = r; s.ct0 = ct0; s.ct1 = ct0 + (int)take; s.slot = (int)(k - kf);
    p += take;
    return true;
  }
};

// Partial slots of the persistent NEG walk that can hold sums of one row tile: G CTAs walk the row_tiles x col_tiles
// pairs in contiguous ranges of U = P / G >= 1 pairs, so a row tile's col_tiles pairs meet at most col_tiles / U + 2 CTAs.
__host__ __device__ __forceinline__ long long neg_slot_bound(long long row_tiles, long long col_tiles, int grid) {
  const long long P = row_tiles * col_tiles;
  const long long U = P / (grid > 1 ? grid : 1);
  return col_tiles / (U > 1 ? U : 1) + 2;
}

// Row prologue of the POS sweeps: the sum over negatives of `row` = fixed-order sum of the NEG sweep's partial slots
// (unwritten slots hold 0) + the analytic zero tail of the flattened bank (Q3).  `publish`: the CTA of split 0 writes
// (m, Neg) to the row statistics for the backward.
__device__ __forceinline__ float pos_row_neg(const TcArgs& a, const float* partials, int A, int col_tiles, int row,
                                             int rcls, float m2, bool publish, float* rowstats_out) {
  const int64_t stride = (int64_t)a.slots * a.a_pad;
  const int used = (int)min((long long)a.slots, neg_slot_bound((A + BM - 1) / BM, col_tiles, a.neg_grid));
  float n = 0.f;
#pragma unroll 8
  for (int pslot = 0; pslot < used; ++pslot) n += __ldcg(partials + stride + (int64_t)pslot * a.a_pad + row);
  if (a.tail_count > 0 && rcls != 0) {
    // the zero tail takes part in the a10 selection with the key of +0.0
    const float wt = a.tk_sel ? topk_weight(KEY_ZERO, a.tk_sel[row], __uint_as_float(a.tk_sel[a.a_rows + row])) : 1.f;
    n += wt * (float)a.tail_count * ptx::ex2_approx(-m2);
  }
  if (publish && rowstats_out != nullptr) {
    rowstats_out[row] = m2 * LN2;
    rowstats_out[a.a_rows + row] = n;
  }
  return n;
}

// Barriers of a ring pipeline (full / empty per stage, a_full / a_empty for the operand that stays), by one thread.
template <int STAGES_, class Smem>
__device__ __forceinline__ void init_ring_barriers(Smem& sm, const CUtensorMap* tm0, const CUtensorMap* tm1) {
  ptx::prefetch_tmap(tm0);
  ptx::prefetch_tmap(tm1);
  for (int s = 0; s < STAGES_; ++s) { ptx::mbar_init(&sm.full[s], 1); ptx::mbar_init(&sm.empty[s], CONSUMER_WARPS); }
  ptx::mbar_init(&sm.a_full, 1);
  ptx::mbar_init(&sm.a_empty, CONSUMER_WARPS);
  ptx::fence_barrier_init();
}

// The TMA producer of a ring pipeline, one work item with tiles [t0, t1) (t1 > t0): once the previous item's MMAs have
// retired, the operand that stays (NKB boxes of FIXED_KB bytes from row `fixed_row`, into sm.a), then NKB boxes of
// RING_KB bytes per tile of TILE_ROWS rows through the ring (sm.c).  `item` counts the items loaded so far.
struct ProducerState { uint32_t stage = 0, phase = 0; int item = 0; };
template <int STAGES_, int FIXED_KB, int RING_KB, int TILE_ROWS, class Smem>
__device__ __forceinline__ void produce_item(Smem& sm, ProducerState& p, const CUtensorMap* tm_fixed,
                                             const CUtensorMap* tm_ring, int fixed_row, int t0, int t1) {
  if (p.item > 0) ptx::mbar_wait(&sm.a_empty, (p.item - 1) & 1);
  ptx::mbar_arrive_expect_tx(&sm.a_full, NKB * FIXED_KB);
  for (int kb = 0; kb < NKB; ++kb) ptx::tma_load_2d(sm.a + kb * FIXED_KB, tm_fixed, &sm.a_full, kb * BK, fixed_row);
  for (int t = t0; t < t1; ++t) {
    for (int kb = 0; kb < NKB; ++kb) {
      ptx::mbar_wait(&sm.empty[p.stage], p.phase ^ 1);
      ptx::mbar_arrive_expect_tx(&sm.full[p.stage], RING_KB);
      ptx::tma_load_2d(sm.c + p.stage * RING_KB, tm_ring, &sm.full[p.stage], kb * BK, t * TILE_ROWS);
      if (++p.stage == STAGES_) { p.stage = 0; p.phase ^= 1; }
    }
  }
  ++p.item;
}

template <int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
k_tc_fwd(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, TcArgs a,
         float* __restrict__ partials, float* __restrict__ rowstats_out) {
  extern __shared__ uint8_t smem_raw[];
  // Rounded through an integer, unlike aligned_smem: the staging buffer is then reached by generic loads and stores,
  // and the NEG sweep at A = 65536 x N = 131072 ran 10.49 - 10.68 ms that way against 10.69 - 11.00 ms with LDS / STS
  // (H100 SXM, 700 W).
  SmemLayout& sm = *reinterpret_cast<SmemLayout*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int A = a.plan ? min(a.plan[PCL_PLAN_A], a.a_rows) : a.a_rows;
  if (A <= 0) return;
  const int64_t ncols = a.mode == 0 ? (int64_t)A : a.n_cols;
  const int T_all = (int)((ncols + BN - 1) / BN);

  // ---- work list of this CTA (identical in every warp) ----
  SegWalker w0;
  w0.persistent = a.persistent != 0;
  w0.pending = false;
  w0.T = T_all; w0.G = gridDim.x; w0.k = blockIdx.x;
  if (w0.persistent) {
    const int R_live = (A + BM - 1) / BM;
    w0.P = (long long)R_live * T_all;
    // The grid is sized on the host for a_rows; with a device-side plan fewer pairs may be live.  Spreading them over
    // more CTAs than pairs would leave idle CTAs between the working ones, and a CTA's ordinal among those touching a
    // row tile (its partial slot) could then pass the slots the workspace has: the CTAs past P stay idle instead.
    if (w0.G > w0.P) w0.G = (int)w0.P;
    if (blockIdx.x >= w0.G) return;
    w0.p = ((long long)blockIdx.x * w0.P) / w0.G;
    w0.p_end = ((long long)(blockIdx.x + 1) * w0.P) / w0.G;
    if (w0.p >= w0.p_end) return;
  } else {
    const int row0 = blockIdx.x * BM;
    if (row0 >= A) return;
    int t_lo = 0, t_hi = T_all;
    if (MODE == TC_POS && a.mode == 2 && a.sorted && a.cls_start != nullptr) {
      // positives of this row tile live in the columns of its label range (contrast labels are sorted)
      int lo = 0x7fffffff, hi = -1;
      for (int i = lane; i < BM; i += 32) {
        const int r = row0 + i;
        if (r < A) { const int c = a.acls[r]; lo = min(lo, c); hi = max(hi, c); }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
      }
      lo = max(0, min(lo, PCL_MAX_CLASSES - 1));
      hi = max(0, min(hi, PCL_MAX_CLASSES - 1));
      t_lo = a.cls_start[lo] / BN;
      t_hi = (a.cls_start[hi + 1] + BN - 1) / BN;
      if (t_hi < t_lo) t_hi = t_lo;
    }
    if (MODE == TC_POS && a.mode == 0 && a.sorted) {
      // self-contrast with class-grouped anchors: the positives of this row tile are the rows of its classes, one
      // contiguous run [lo, hi) around the tile
      const int last = min(A - 1, row0 + BM - 1);
      const int c_first = a.acls[row0], c_last = a.acls[last];
      int lo = row0, hi = last + 1;
      for (;;) {                                   // warp-parallel run search: 32 rows per probe, no dependent loads
        const int idx = lo - 1 - lane;
        const unsigned m = __ballot_sync(0xffffffffu, idx >= 0 && a.acls[idx] == c_first);
        const int run = (m == 0xffffffffu) ? 32 : __ffs(~m) - 1;
        lo -= run;
        if (run < 32) break;
      }
      for (;;) {
        const int idx = hi + lane;
        const unsigned m = __ballot_sync(0xffffffffu, idx < A && a.acls[idx] == c_last);
        const int run = (m == 0xffffffffu) ? 32 : __ffs(~m) - 1;
        hi += run;
        if (run < 32) break;
      }
      t_lo = lo / BN;
      t_hi = (hi + BN - 1) / BN;
    }
    if (MODE == TC_POS && a.mode == 1) {
      const int last = min(A - 1, row0 + BM - 1);
      int rk_f = class_rank(a.acls[row0], a.K), rk_l = class_rank(a.acls[last], a.K);
      if (rk_l > a.K - 2) rk_l = a.K - 2;
      if (rk_f > rk_l) { t_lo = 0; t_hi = 0; }
      else {
        t_lo = (int)(((int64_t)rk_f * a.R) / BN);
        t_hi = (int)((((int64_t)(rk_l + 1) * a.R) + BN - 1) / BN);
      }
    }
    const int span = t_hi - t_lo;
    const int per = (span + a.splits - 1) / a.splits;
    const int my_lo = t_lo + blockIdx.y * per;
    const int my_hi = min(t_hi, my_lo + per);
    w0.single.r = blockIdx.x; w0.single.ct0 = my_lo; w0.single.ct1 = my_hi > my_lo ? my_hi : my_lo;
    w0.single.slot = blockIdx.y;
    w0.pending = true;
    w0.p = w0.p_end = w0.P = 0;
  }

  // ---- one-time setup ----
  if (warp == PRODUCER_WARP && lane == 0) init_ring_barriers<STAGES>(sm, &tmA, &tmB);
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    // =========================== TMA producer ===========================
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP && lane == 0) {
      SegWalker w = w0;
      Seg sg;
      ProducerState ps;
      while (w.next(sg))
        if (sg.ct1 > sg.ct0) produce_item<STAGES, A_KB_BYTES, B_STAGE_BYTES, BN>(sm, ps, &tmA, &tmB, sg.r * BM, sg.ct0, sg.ct1);
    }
  } else {
    // =========================== consumer warpgroups: wgmma + epilogue ===========================
    ptx::setmaxnreg_inc<CONSUMER_REGS>();
    const int g = threadIdx.x >> 7, t = threadIdx.x & 127;
    const int half = t >> 6;                          // which 128 columns of the 256-column tile
    const int r_in = g * 64 + (t & 63);
    const uint32_t a_base = ptx::smem_u32(sm.a) + g * WG_ROW_BYTES, b_base = ptx::smem_u32(sm.c);
    Ring ring;
    SegWalker w = w0;
    Seg sg;
    int seg_idx = 0;
    while (w.next(sg)) {
      const int row = sg.r * BM + r_in;
      const bool valid = row < A;
      const int rcls = valid ? a.acls[row] : -1;
      const int rdiag = valid ? (a.mode == 0 ? row : (a.diag ? a.diag[row] : -1)) : -1;
      const float m2 = valid ? a.row_m2[row] : 0.f;
      float neg_i = 1.f;
      if (MODE == TC_POS && valid) neg_i = pos_row_neg(a, partials, A, T_all, row, rcls, m2, sg.slot == 0, rowstats_out);
      // a10 selection state of this row: key prefix (H2, H3) / tau key and tie weight (NEGW)
      uint32_t tk_pref = TK_ALL;
      float tk_tw = 0.f;
      uint32_t* tk_hrow = nullptr;
      if (MODE == TC_H1 || MODE == TC_H2 || MODE == TC_H3 || MODE == TC_NEGW) {
        if (valid) {
          if (MODE != TC_H1) tk_pref = a.tk_sel[row];
          if (MODE == TC_NEGW) tk_tw = __uint_as_float(a.tk_sel[a.a_rows + row]);
          tk_hrow = a.tk_hist + (int64_t)row * TK_BINS;
        }
      }
      float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;     // NEG: 4 partial sums; POS: possum2, s, cnt
      int nlab_lo[4], nlab_hi[4];                              // first / last label of the 4 chunks of the next tile
      chunk_labels<4>(a, sg.ct0 * BN + half * (BN / 2), sg.ct0 < sg.ct1 && a.sorted, ncols, nlab_lo, nlab_hi);
      if (sg.ct1 > sg.ct0) ptx::mbar_wait(&sm.a_full, seg_idx & 1);
      for (int ct = sg.ct0; ct < sg.ct1; ++ct) {
        float acc[128];
        ring_mma<STAGES, B_STAGE_BYTES, false>(acc, a_base, A_KB_BYTES, b_base, sm.full, sm.empty, ring, lane);
        if (ct + 1 == sg.ct1 && lane == 0) ptx::mbar_arrive(&sm.a_empty);     // last MMA of the segment retired
        const int col0 = ct * BN + half * (BN / 2);
        // Per 32-column chunk: if the chunk is complete and of one class (sorted contrast set) every row treats it as
        // all-negative or all-positive without a per-element test.  Mixed chunks (a class boundary, the ragged end,
        // self-contrast) fetch one label per lane and broadcast it with warp shuffles — no dependent loads.
        // (labels were fetched one tile ahead: the loads are in flight while the previous tile is processed)
        int clab[4];
        bool cuni[4];
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
          const int cb = col0 + ch * 32;
          clab[ch] = nlab_lo[ch];
          cuni[ch] = a.sorted && cb + 32 <= ncols && nlab_lo[ch] == nlab_hi[ch];
        }
        if (ct + 1 < sg.ct1) {
          chunk_labels<4>(a, (ct + 1) * BN + half * (BN / 2), a.sorted != 0, ncols, nlab_lo, nlab_hi);
        }
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
          // chunk ch of both column halves -> staging buffer -> this thread's row, 32 columns
          frag_store_cols<4>(acc, 4 * ch, &sm.stage[g][0][0][0], SPITCH, t);
          frag_store_cols<4>(acc, 16 + 4 * ch, &sm.stage[g][1][0][0], SPITCH, t);
          ptx::bar_sync(2 + g, 128);
          uint32_t v[32];
          load_row32(&sm.stage[g][half][t & 63][0], v);
          ptx::bar_sync(2 + g, 128);
          const int cb = col0 + ch * 32;
          const bool uniform = cuni[ch];
          const int ulab = clab[ch];
          if (MODE == TC_DUMP) {
            // partials doubles as the dump buffer: [a_pad][ld], ld = column tiles * BN
            const int64_t ld = (int64_t)T_all * BN;
#pragma unroll
            for (int j = 0; j < 32; ++j) partials[(int64_t)row * ld + cb + j] = __uint_as_float(v[j]);
          } else if (MODE == TC_H1 || MODE == TC_H2 || MODE == TC_H3 || MODE == TC_NEGW) {
            // a10: every NEGATIVE logit of the row goes through its sortable key
            const int mylab = uniform ? ulab : ((cb + lane < ncols) ? col_label(a, cb + lane) : -2);
            if (MODE == TC_NEGW) {
              // branch-free: one ex2 per logit like the plain NEG sweep, times the selection weight (0, 1 or the tie share);
              // a branch on w > 0 diverged on almost every element (some lane of the warp keeps it): 568 us vs 86 for NEG
#pragma unroll
              for (int j = 0; j < 32; j += 2) {
                const int l0 = uniform ? ulab : __shfl_sync(0xffffffffu, mylab, j);
                const int l1 = uniform ? ulab : __shfl_sync(0xffffffffu, mylab, j + 1);
                const float x0 = __fmul_rn(__uint_as_float(v[j]), a.k1), x1 = __fmul_rn(__uint_as_float(v[j + 1]), a.k1);
                const float w0 = (valid && l0 != -2 && l0 != rcls) ? topk_weight(sortable_key(x0), tk_pref, tk_tw) : 0.f;
                const float w1 = (valid && l1 != -2 && l1 != rcls) ? topk_weight(sortable_key(x1), tk_pref, tk_tw) : 0.f;
                const float e0 = ptx::ex2_approx(x0 - m2), e1 = ptx::ex2_approx(x1 - m2);
                acc0 = fmaf(w0, w0 > 0.f ? e0 : 0.f, acc0);       // (select, not multiply: an excluded logit may overflow)
                acc1 = fmaf(w1, w1 > 0.f ? e1 : 0.f, acc1);
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                const int lj = uniform ? ulab : __shfl_sync(0xffffffffu, mylab, j);
                if (valid && lj != -2 && lj != rcls) {
                  const float x = __fmul_rn(__uint_as_float(v[j]), a.k1);
                  const uint32_t key = sortable_key(x);
                  if (MODE == TC_H1) {
                    atomicAdd(tk_hrow + (key >> 21), 1u);
                  } else if (MODE == TC_H2) {
                    if ((key >> 21) == tk_pref) atomicAdd(tk_hrow + ((key >> 10) & 0x7FFu), 1u);
                  } else {
                    if ((key >> 10) == tk_pref) atomicAdd(tk_hrow + (key & 0x3FFu), 1u);
                  }
                }
              }
            }
          } else if (MODE == TC_NEG) {
            if (uniform) {
              if (valid && ulab != rcls) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                  acc0 += ptx::ex2_approx(fmaf(__uint_as_float(v[j + 0]), a.k1, -m2));
                  acc1 += ptx::ex2_approx(fmaf(__uint_as_float(v[j + 1]), a.k1, -m2));
                  acc2 += ptx::ex2_approx(fmaf(__uint_as_float(v[j + 2]), a.k1, -m2));
                  acc3 += ptx::ex2_approx(fmaf(__uint_as_float(v[j + 3]), a.k1, -m2));
                }
              }
            } else {
              const int mylab = (cb + lane < ncols) ? col_label(a, cb + lane) : -2;
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                const int lj = __shfl_sync(0xffffffffu, mylab, j);
                const float e = ptx::ex2_approx(fmaf(__uint_as_float(v[j]), a.k1, -m2));
                acc0 += (valid && lj != -2 && lj != rcls) ? e : 0.f;
              }
            }
          } else {
            if (uniform) {
              if (valid && ulab == rcls) {
                const bool has_diag = rdiag >= cb && rdiag < cb + 32;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                  const float x = fmaf(__uint_as_float(v[j]), a.k1, -m2);
                  const float t = ptx::ex2_approx(x) + neg_i;
                  const float keep = (has_diag && cb + j == rdiag) ? 0.f : 1.f;
                  acc0 += keep * (x - ptx::lg2_approx(t));
                  acc1 += keep * ptx::rcp_approx(t);
                  acc2 += keep;
                }
              }
            } else {
              const int mylab = (cb + lane < ncols) ? col_label(a, cb + lane) : -2;
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                const int lj = __shfl_sync(0xffffffffu, mylab, j);
                if (valid && lj == rcls && cb + j != rdiag) {
                  const float x = fmaf(__uint_as_float(v[j]), a.k1, -m2);
                  const float t = ptx::ex2_approx(x) + neg_i;
                  acc0 += x - ptx::lg2_approx(t);
                  acc1 += ptx::rcp_approx(t);
                  acc2 += 1.f;
                }
              }
            }
          }
        }
      }
      if (sg.ct1 > sg.ct0) ++seg_idx;
      // ---- combine the two column halves, write the partials of this segment ----
      if (MODE != TC_DUMP && MODE != TC_H1 && MODE != TC_H2 && MODE != TC_H3) {
        if (MODE == TC_NEG || MODE == TC_NEGW) {
          sm.comb[0][half][r_in] = (acc0 + acc1) + (acc2 + acc3);
        } else {
          sm.comb[0][half][r_in] = acc0 * LN2;
          sm.comb[1][half][r_in] = acc1;
          sm.comb[2][half][r_in] = acc2;
        }
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
        if (half == 0) {
          const int64_t o = (int64_t)sg.slot * a.a_pad + row;
          const int64_t stride = (int64_t)a.slots * a.a_pad;
          if (MODE == TC_NEG || MODE == TC_NEGW) {
            partials[0 * stride + o] = m2 * LN2;                             // stabiliser in natural-log units
            partials[1 * stride + o] = sm.comb[0][0][r_in] + sm.comb[0][1][r_in];
          } else {
            partials[2 * stride + o] = sm.comb[0][0][r_in] + sm.comb[0][1][r_in];
            partials[3 * stride + o] = sm.comb[1][0][r_in] + sm.comb[1][1][r_in];
            partials[4 * stride + o] = sm.comb[2][0][r_in] + sm.comb[2][1][r_in];
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");       // comb reusable by the next segment
      }
    }
  }
}

// =====================================================================================================
// POS sweep of the bank mode for SMALL anchor sets, transposed: the bank's column tile is the M operand (accumulator
// row = bank column, 64 per consumer warpgroup), a block of <= 64 anchors of ONE class the N operand.  The positives of
// an anchor are the R columns of its class, so the work list is (class, anchor block, column split) and every element
// the epilogue touches is a positive: every consumer thread works, whatever the class mix of the anchors.  (The
// row-tile POS sweep above computes [128 anchors x 256 columns] tiles in which only the rows of the tile's class do
// anything: with ~53 anchors per class — configs[2] — one or two of the eight consumer warps would carry a CTA.)
// Per-anchor sums are reduced across the bank columns once per work item.
// Anchors must be in class-rank order (bank mode's contract, like the row-tile sweep's [rk_f, rk_l] range).
// =====================================================================================================
constexpr int PT_NB = 64;                          // anchors per block (N of the MMA)
constexpr int PT_BM = 128;                         // bank columns per tile (M of the MMA)
constexpr int PT_A_KB = PT_NB * BK * 2;            // 8 KB: [64 anchors x 64 K] box
constexpr int PT_C_KB = PT_BM * BK * 2;            // 16 KB: [128 columns x 64 K] box
constexpr int PT_STAGES = 8;                       // K-block stages of the bank stream (2 tiles in flight)
static_assert(PT_BM == 2 * 64, "one M64 wgmma per consumer warpgroup");
constexpr int PT_MAX_ROWS = 4096;                  // class-boundary scan of the prologue

constexpr int PT_MAX_BLOCKS = PT_MAX_ROWS / PT_NB + PCL_MAX_CLASSES;      // blocks of <= 64 anchors of one class

struct SmemPosT {
  uint8_t a[NKB * PT_A_KB];                        // 32 KB
  uint8_t c[PT_STAGES * PT_C_KB];                  // 128 KB
  float stage[2][64][PT_NB + 4];                   // [warpgroup][bank column][anchor]: the accumulator, row view
  uint64_t full[PT_STAGES], empty[PT_STAGES], a_full, a_empty;
  int rk_first[PCL_MAX_CLASSES], rk_cnt[PCL_MAX_CLASSES];
  // work list: anchor blocks (first row, rows, class rank), exclusive prefix of their column tiles, blocks without tiles
  int blk_r0[PT_MAX_BLOCKS], blk_rk[PT_MAX_BLOCKS], tile_pref[PT_MAX_BLOCKS + 1], zlist[PT_MAX_BLOCKS];
  short blk_nv[PT_MAX_BLOCKS];
  int total_blocks, n_zero, P, U;
  float4 par[PT_NB];                               // per anchor of the block: m2, Neg, diag column (int bits), -
  float comb[2][4][32][2];                         // [anchor half][column quarter][anchor][possum2, s]
};
static_assert(sizeof(SmemPosT) + 1024 <= 227 * 1024, "shared memory of one H100 block");

// One segment = consecutive column tiles [t0, t1) of one anchor block; its partial sums go to slot `split`; the block
// is covered by `nslots` segments (of consecutive CTAs).
struct PosItem { int r0, nv, t0, t1, c_lo, c_hi, split, nslots; };

// All tile units (block, tile) form one list of P entries; CTA k owns units [k U, (k+1) U) — a balanced walk whatever
// the class mix (K = 171 classes: 171 blocks on 132 CTAs would otherwise make 39 CTAs do twice the work).  Every role
// (TMA producer / consumer warpgroups) walks the same segments.  Blocks without tiles (class-0 anchors: their positives are the
// analytic zero tail, k_finalize) are dealt round-robin and only write their rows.
struct PosWalk {
  int u, u1, blk, z, k, G;
  __device__ __forceinline__ void init(const SmemPosT& sm, int cta, int grid) {
    k = cta; G = grid;
    u = min(sm.P, cta * sm.U); u1 = min(sm.P, u + sm.U);
    blk = 0; z = cta;
  }
  __device__ __forceinline__ bool next(const SmemPosT& sm, const TcArgs& a, PosItem& it) {
    if (u < u1) {
      while (sm.tile_pref[blk + 1] <= u) ++blk;
      const int b0 = sm.tile_pref[blk], b1 = sm.tile_pref[blk + 1];
      const int e = min(u1, b1);
      const int rk = sm.blk_rk[blk];
      it.r0 = sm.blk_r0[blk]; it.nv = sm.blk_nv[blk];
      it.c_lo = rk * a.R; it.c_hi = it.c_lo + a.R;
      const int t_lo = it.c_lo / PT_BM;
      it.t0 = t_lo + (u - b0); it.t1 = t_lo + (e - b0);
      it.split = k - b0 / sm.U;
      it.nslots = (b1 - 1) / sm.U - b0 / sm.U + 1;
      u = e;
      return true;
    }
    if (z < sm.n_zero) {
      const int b = sm.zlist[z];
      z += G;
      it.r0 = sm.blk_r0[b]; it.nv = sm.blk_nv[b];
      it.c_lo = it.c_hi = 0; it.t0 = it.t1 = 0; it.split = 0; it.nslots = 0;
      return true;
    }
    return false;
  }
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
k_tc_pos_t(const __grid_constant__ CUtensorMap tmA64, const __grid_constant__ CUtensorMap tmC128, TcArgs a,
           float* __restrict__ partials, float* __restrict__ rowstats_out) {
  extern __shared__ uint8_t smem_raw[];
  SmemPosT& sm = aligned_smem<SmemPosT>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int A = a.plan ? min(a.plan[PCL_PLAN_A], a.a_rows) : a.a_rows;
  if (A <= 0) return;

  // ---- class runs of the anchors (class-rank order) -> blocks of <= 64 anchors, S column splits per block ----
  for (int i = threadIdx.x; i < PCL_MAX_CLASSES; i += blockDim.x) { sm.rk_first[i] = 0; sm.rk_cnt[i] = 0; }
  __syncthreads();
  for (int r = threadIdx.x; r < A; r += blockDim.x) {
    const int rk = min(max(class_rank(a.acls[r], a.K), 0), PCL_MAX_CLASSES - 1);
    if (r == 0 || class_rank(a.acls[r - 1], a.K) != class_rank(a.acls[r], a.K)) sm.rk_first[rk] = r;
    atomicAdd(&sm.rk_cnt[rk], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int nb = 0, nz = 0, P = 0, tmax = 1;
    for (int rk = 0; rk < a.K && rk < PCL_MAX_CLASSES; ++rk) {
      const int cnt = sm.rk_cnt[rk];
      int tiles = 0;
      if (rk <= a.K - 2) {
        const int c_lo = rk * a.R;
        tiles = (c_lo + a.R + PT_BM - 1) / PT_BM - c_lo / PT_BM;
      }
      for (int b = 0; b * PT_NB < cnt && nb < PT_MAX_BLOCKS; ++b) {
        sm.blk_r0[nb] = sm.rk_first[rk] + b * PT_NB;
        sm.blk_nv[nb] = (short)min(PT_NB, cnt - b * PT_NB);
        sm.blk_rk[nb] = rk;
        sm.tile_pref[nb] = P;
        P += tiles;
        if (tiles == 0) sm.zlist[nz++] = nb;
        tmax = max(tmax, tiles);
        ++nb;
      }
    }
    sm.tile_pref[nb] = P;
    sm.total_blocks = nb; sm.n_zero = nz; sm.P = P;
    // units per CTA: even share, but a block must not be cut into more segments than there are partial slots
    int U = (P + (int)gridDim.x - 1) / (int)gridDim.x;
    const int u_slots = a.splits >= 2 ? (tmax + a.splits - 2) / (a.splits - 1) : max(P, 1);
    sm.U = max(1, max(U, u_slots));
    init_ring_barriers<PT_STAGES>(sm, &tmA64, &tmC128);
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    // =========================== TMA producer ===========================
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP && lane == 0) {
      ProducerState ps;
      PosWalk w;
      PosItem it;
      w.init(sm, blockIdx.x, gridDim.x);
      while (w.next(sm, a, it))
        if (it.t1 > it.t0) produce_item<PT_STAGES, PT_A_KB, PT_C_KB, PT_BM>(sm, ps, &tmA64, &tmC128, it.r0, it.t0, it.t1);
    }
  } else {
    // =========================== consumer warpgroups: wgmma (M = 64 bank columns each, N = 64 anchors) + epilogue ====
    ptx::setmaxnreg_inc<CONSUMER_REGS>();
    const int g = threadIdx.x >> 7, t = threadIdx.x & 127;
    const int quarter = g * 2 + ((t & 63) >> 5);      // which 32 bank columns of the 128-column tile
    const int ahalf = t >> 6;                         // which 32 anchors of the block
    const int et = threadIdx.x;                       // 0..255 within the consumer group
    const uint32_t a_base = ptx::smem_u32(sm.a), c_base = ptx::smem_u32(sm.c) + g * WG_ROW_BYTES;
    const int64_t stride = (int64_t)a.slots * a.a_pad;
    Ring ring;
    int seq = 0;
    PosWalk w;
    PosItem it;
    w.init(sm, blockIdx.x, gridDim.x);
    while (w.next(sm, a, it)) {
      // ---- per-anchor constants of the block (the row prologue of the row-tile sweep, one thread per anchor) ----
      if (et < PT_NB) {
        float4 pr = make_float4(0.f, 1.f, __int_as_float(-1), 0.f);
        if (et < it.nv && it.r0 + et < A) {
          const int row = it.r0 + et;
          const float m2 = a.row_m2[row];
          const int col_tiles = (int)((a.n_cols + BN - 1) / BN);
          const float ng = pos_row_neg(a, partials, A, col_tiles, row, a.acls[row], m2, it.split == 0, rowstats_out);
          pr = make_float4(m2, ng, __int_as_float(a.diag ? a.diag[row] : -1), 0.f);
        }
        sm.par[et] = pr;
      }
      asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
      float acc0[32], acc1[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
      const int nvh = min(32, max(0, it.nv - ahalf * 32));                  // valid anchors of this warp's half
      if (it.t1 > it.t0) ptx::mbar_wait(&sm.a_full, seq & 1);
      for (int tl = it.t0; tl < it.t1; ++tl) {
        float acc[32];
        ring_mma<PT_STAGES, PT_C_KB, true>(acc, a_base, PT_A_KB, c_base, sm.full, sm.empty, ring, lane);
        if (tl + 1 == it.t1 && lane == 0) ptx::mbar_arrive(&sm.a_empty);     // last MMA of the block retired
        frag_store_cols<8>(acc, 0, &sm.stage[g][0][0], PT_NB + 4, t);
        ptx::bar_sync(2 + g, 128);
        uint32_t v[32];
        load_row32(&sm.stage[g][t & 63][ahalf * 32], v);
        ptx::bar_sync(2 + g, 128);
        const int col = tl * PT_BM + quarter * 32 + lane;
        const bool colkeep = col >= it.c_lo && col < it.c_hi;
        // groups of 8 anchors behind ONE warp-uniform test: inside a group the 8 LDS -> FMA -> EX2 -> LG2 / RCP chains
        // are independent and interleave (a test per anchor makes 32 basic blocks, i.e. 32 serial MUFU chains per
        // tile).  Anchors
        // past the block's end inside a group carry neutral constants (m2 = 0, Neg = 1) and are never written.
#pragma unroll
        for (int i0 = 0; i0 < 32; i0 += 8) {
          if (i0 < nvh) {
#pragma unroll
            for (int i = i0; i < i0 + 8; ++i) {
              const float4 pr = sm.par[ahalf * 32 + i];                       // broadcast read
              const float x = fmaf(__uint_as_float(v[i]), a.k1, -pr.x);
              const float tt = ptx::ex2_approx(x) + pr.y;
              const bool keep = colkeep && col != __float_as_int(pr.z);
              acc0[i] += keep ? x - ptx::lg2_approx(tt) : 0.f;
              acc1[i] += keep ? ptx::rcp_approx(tt) : 0.f;
            }
          }
        }
      }
      if (it.t1 > it.t0) ++seq;
      // ---- sum over the 128 lanes (columns): butterfly inside the warp, then the 4 quarters through shared memory ----
#pragma unroll
      for (int i = 0; i < 32; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          acc0[i] += __shfl_xor_sync(0xffffffffu, acc0[i], o);
          acc1[i] += __shfl_xor_sync(0xffffffffu, acc1[i], o);
        }
        if (lane == i) { sm.comb[ahalf][quarter][i][0] = acc0[i]; sm.comb[ahalf][quarter][i][1] = acc1[i]; }
      }
      asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
      if (et < it.nv && it.r0 + et < A) {
        const int h = et >> 5, i = et & 31, row = it.r0 + et;
        const float ps = (sm.comb[h][0][i][0] + sm.comb[h][1][i][0]) + (sm.comb[h][2][i][0] + sm.comb[h][3][i][0]);
        const float ss = (sm.comb[h][0][i][1] + sm.comb[h][1][i][1]) + (sm.comb[h][2][i][1] + sm.comb[h][3][i][1]);
        // positives counted analytically: the class columns inside this split's tile range, minus the masked (i, diag_i)
        const int lo = max(it.c_lo, it.t0 * PT_BM), hi = min(it.c_hi, it.t1 * PT_BM);
        const int dg = __float_as_int(sm.par[et].z);
        const int cnt = max(0, hi - lo) - ((dg >= lo && dg < hi) ? 1 : 0);
        const int64_t o = (int64_t)it.split * a.a_pad + row;
        partials[2 * stride + o] = ps * LN2;
        partials[3 * stride + o] = ss;
        partials[4 * stride + o] = (float)cnt;
        if (it.split == 0) {                                                  // slots no segment of this block writes: k_finalize sums a.splits of them
          for (int sl = it.nslots; sl < a.splits; ++sl) {
            const int64_t oz = (int64_t)sl * a.a_pad + row;
            partials[2 * stride + oz] = 0.f; partials[3 * stride + oz] = 0.f; partials[4 * stride + oz] = 0.f;
          }
        }
      }
      asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");       // par / comb reusable by the next item
    }
  }
}

// =====================================================================================================
// Backward: dA = G . C / T with G formed on the fly (closed form, SURVEY appendix A) — FlashAttention-backward
// shaped, per consumer warpgroup (64 anchor rows): wgmma 1 S = A.C^T (64 x 64 tile, K = 256) -> epilogue turns S into
// the bf16 gradient tile G in shared memory (128B-swizzled K-major) -> wgmma 2 dA(64 x 256, registers, across the whole
// column sweep) += G . C, where the SAME shared-memory contrast tile is re-read as an MN-major B operand.
// =====================================================================================================
constexpr int BNB = 64;                           // columns per tile in the backward sweep
constexpr int C_KB_BYTES = BNB * BK * 2;          // 8 KB: one [64 x 64] box
constexpr int C_STAGE_BYTES = NKB * C_KB_BYTES;   // 32 KB: the full [64 x 256] tile
constexpr int G_BYTES = BM * BNB * 2;             // 16 KB
constexpr int BWD_STAGES = 3;

struct SmemBwd {
  uint8_t a[NKB * A_KB_BYTES];                    // 64 KB
  uint8_t c[BWD_STAGES * C_STAGE_BYTES];          // 96 KB
  uint8_t g[G_BYTES];                             // 16 KB
  float stage[2][64][BNB + 4];                    // [warpgroup][row][column]: S, row view
  uint64_t a_full, c_full[BWD_STAGES], c_empty[BWD_STAGES];
};
static_assert(sizeof(SmemBwd) + 1024 <= 227 * 1024, "shared memory of one H100 block");

struct TcBwdArgs {
  TcArgs t;
  const float* rowstats;       // m, neg, possum, s, npos, row_loss (a_rows each)
  float rs_scale;              // (T / bT) / A_live is applied per row: c_i = rs_scale' / npos_i; here T/bT
  int nan_safe;
};

template <bool TOPK>
__global__ void __launch_bounds__(NUM_THREADS, 1)
k_tc_bwd(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmC, TcBwdArgs ba,
         float* __restrict__ dpartials) {
  extern __shared__ uint8_t smem_raw[];
  SmemBwd& sm = aligned_smem<SmemBwd>(smem_raw);
  const TcArgs& a = ba.t;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int A = a.plan ? min(a.plan[PCL_PLAN_A], a.a_rows) : a.a_rows;
  const int row0 = blockIdx.x * BM;
  if (row0 >= A) return;
  const int split = blockIdx.y;
  const int64_t ncols = a.mode == 0 ? (int64_t)A : a.n_cols;
  const int t_hi = (int)((ncols + BNB - 1) / BNB);
  // Column tiles are dealt round-robin to the splits (tile = split + it * splits): the tiles that hold a row tile's
  // positives (2 MUFU ops per logit, divergent rows) are spread over all its CTAs instead of landing on two or three
  // of them (contiguous ranges left 30 % of the SM time idle behind the slowest CTAs).
  const int my_lo = split, tstep = a.splits;
  const int ntiles = t_hi > split ? (t_hi - split + a.splits - 1) / a.splits : 0;

  if (warp == PRODUCER_WARP && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmC);
    ptx::mbar_init(&sm.a_full, 1);
    for (int s = 0; s < BWD_STAGES; ++s) { ptx::mbar_init(&sm.c_full[s], 1); ptx::mbar_init(&sm.c_empty[s], CONSUMER_WARPS); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP && lane == 0 && ntiles > 0) {
      ptx::mbar_arrive_expect_tx(&sm.a_full, NKB * A_KB_BYTES);
      for (int kb = 0; kb < NKB; ++kb) ptx::tma_load_2d(sm.a + kb * A_KB_BYTES, &tmA, &sm.a_full, kb * BK, row0);
      for (int it = 0; it < ntiles; ++it) {
        const int stage = it % BWD_STAGES, phase = (it / BWD_STAGES) & 1;
        ptx::mbar_wait(&sm.c_empty[stage], phase ^ 1);
        ptx::mbar_arrive_expect_tx(&sm.c_full[stage], C_STAGE_BYTES);
        for (int kb = 0; kb < NKB; ++kb)
          ptx::tma_load_2d(sm.c + stage * C_STAGE_BYTES + kb * C_KB_BYTES, &tmC, &sm.c_full[stage], kb * BK,
                           (my_lo + it * tstep) * BNB);
      }
    }
    return;
  }
  // =========================== consumer warpgroups: wgmma 1, epilogue, wgmma 2 ===========================
  ptx::setmaxnreg_inc<CONSUMER_REGS>();
  const int g = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int half = t >> 6;                        // which 32 columns of the 64-column tile
  const int r_in = g * 64 + (t & 63);
  const int row = row0 + r_in;
  const bool valid = row < A;
  const float* st = ba.rowstats;
  const int rcls = valid ? a.acls[row] : -1;
  const int rdiag = valid ? (a.mode == 0 ? row : (a.diag ? a.diag[row] : -1)) : -1;
  const float m2 = valid ? a.row_m2[row] : 0.f;
  const float neg_i = valid ? st[a.a_rows + row] : 1.f;
  const float s_i = valid ? st[3 * a.a_rows + row] : 0.f;
  float c_i = 0.f;
  if (valid) {
    const float np = st[4 * a.a_rows + row];
    c_i = ba.rs_scale / ((float)A * np);
    if (ba.nan_safe && !(np > 0.f)) c_i = 0.f;
  }
  const float cs_i = c_i * s_i;
  const float cn_i = -c_i * neg_i;
  // a10: selection weights on the negatives (tau key, tie weight; pcl_topk.cuh); key = rn(s * k1) as in the forward
  uint32_t tk_tau = 0u;
  float tk_tw = 1.f;
  if (TOPK && valid) { tk_tau = a.tk_sel[row]; tk_tw = __uint_as_float(a.tk_sel[a.a_rows + row]); }
  const uint32_t a_base = ptx::smem_u32(sm.a) + g * WG_ROW_BYTES, c_base = ptx::smem_u32(sm.c);
  const uint32_t g_base = ptx::smem_u32(sm.g) + g * WG_ROW_BYTES;
  uint8_t* g_row = sm.g + r_in * 128;             // + swizzled 16-byte chunk
  float dacc[128];                                // dA of the warpgroup's 64 rows x 256 features
#pragma unroll
  for (int i = 0; i < 128; ++i) dacc[i] = 0.f;
  int nlab_lo[1], nlab_hi[1];
  chunk_labels<1>(a, my_lo * BNB + half * 32, ntiles > 0 && a.sorted && a.mode != 0, (int64_t)ncols, nlab_lo, nlab_hi);
  if (ntiles > 0) ptx::mbar_wait(&sm.a_full, 0);
  for (int it = 0; it < ntiles; ++it) {
    const int ct = my_lo + it * tstep;
    const int stage = it % BWD_STAGES, phase = (it / BWD_STAGES) & 1;
    const int cb = ct * BNB + half * 32;
    const int clab = nlab_lo[0];
    const bool cuni = a.sorted && a.mode != 0 && cb + 32 <= (int)ncols && nlab_lo[0] == nlab_hi[0];
    if (it + 1 < ntiles) {                         // labels of the next tile: loads fly while this tile is processed
      chunk_labels<1>(a, (ct + tstep) * BNB + half * 32, a.sorted && a.mode != 0, (int64_t)ncols, nlab_lo, nlab_hi);
    }
    // ---- wgmma 1: S = A . C^T ----
    ptx::mbar_wait(&sm.c_full[stage], phase);
    const uint32_t c_stage = c_base + stage * C_STAGE_BYTES;
    {
      float sacc[32];
      ptx::wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t da = ptx::make_desc_kmajor_sw128(a_base + kb * A_KB_BYTES + k * 32);
          const uint64_t dc = ptx::make_desc_kmajor_sw128(c_stage + kb * C_KB_BYTES + k * 32);
          ptx::wgmma_m64n64k16<0>(sacc, da, dc, (kb | k) != 0 ? 1u : 0u);
        }
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_operands(sacc);
      frag_store_cols<8>(sacc, 0, &sm.stage[g][0][0], BNB + 4, t);
    }
    ptx::bar_sync(2 + g, 128);
    uint32_t v[32];
    load_row32(&sm.stage[g][t & 63][half * 32], v);
    // ---- epilogue: the gradient tile G of this thread's row, 32 columns ----
    float gv[32];
    if (cuni && clab != rcls) {
      // all-negative chunk: G = c S e   (cs_i == 0 for rows beyond A)
      if (TOPK) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float x = __fmul_rn(__uint_as_float(v[j]), a.k1);
          gv[j] = cs_i * topk_weight(sortable_key(x), tk_tau, tk_tw) * ptx::ex2_approx(x - m2);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) gv[j] = cs_i * ptx::ex2_approx(fmaf(__uint_as_float(v[j]), a.k1, -m2));
      }
    } else if (cuni) {
      // all-positive chunk: G = -c Neg / (e + Neg), zero on the masked (i,i) column
      const bool has_diag = rdiag >= cb && rdiag < cb + 32;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float gpos = cn_i * ptx::rcp_approx(ptx::ex2_approx(fmaf(__uint_as_float(v[j]), a.k1, -m2)) + neg_i);
        gv[j] = (has_diag && cb + j == rdiag) ? 0.f : gpos;
      }
    } else if (a.mode != 0) {
      // mixed chunk: one label per lane, broadcast with shuffles
      const int mylab = (cb + lane < (int)ncols) ? col_label(a, cb + lane) : -2;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int lj = __shfl_sync(0xffffffffu, mylab, j);
        const float xq = __fmul_rn(__uint_as_float(v[j]), a.k1);
        const float e = TOPK ? ptx::ex2_approx(xq - m2) : ptx::ex2_approx(fmaf(__uint_as_float(v[j]), a.k1, -m2));
        const float gneg = TOPK ? cs_i * e * topk_weight(sortable_key(xq), tk_tau, tk_tw) : cs_i * e;
        const float gpos = (cb + j == rdiag) ? 0.f : cn_i * ptx::rcp_approx(e + neg_i);
        gv[j] = (!valid || lj == -2) ? 0.f : (lj == rcls ? gpos : gneg);
      }
    } else {
      // self-contrast: every column is an anchor too -> H = G + G^T needs the column's statistics; lane L holds
      // those of column cb + L and they are broadcast per element
      const int cj = cb + lane;
      const bool cok = cj < (int)ncols;
      const int mylab = cok ? a.acls[cj] : -2;
      float my_m2 = 0.f, my_neg = 1.f, my_cs = 0.f, my_cn = 0.f;
      uint32_t my_tau = 0u;
      float my_tw = 1.f;
      if (TOPK && cok) { my_tau = a.tk_sel[cj]; my_tw = __uint_as_float(a.tk_sel[a.a_rows + cj]); }
      if (cok) {
        const float np_j = st[4 * a.a_rows + cj];
        float c_j = ba.rs_scale / ((float)A * np_j);
        if (ba.nan_safe && !(np_j > 0.f)) c_j = 0.f;
        my_m2 = a.row_m2[cj];
        my_neg = st[a.a_rows + cj];
        my_cs = c_j * st[3 * a.a_rows + cj];
        my_cn = -c_j * my_neg;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int lj = __shfl_sync(0xffffffffu, mylab, j);
        const float m2j = __shfl_sync(0xffffffffu, my_m2, j);
        const float negj = __shfl_sync(0xffffffffu, my_neg, j);
        const float csj = __shfl_sync(0xffffffffu, my_cs, j);
        const float cnj = __shfl_sync(0xffffffffu, my_cn, j);
        const float x = __fmul_rn(__uint_as_float(v[j]), a.k1);
        const float e = ptx::ex2_approx(x - m2);
        const float e2 = ptx::ex2_approx(x - m2j);
        const bool same = lj == rcls;
        const bool diag = (cb + j == rdiag);
        float wi = 1.f, wj = 1.f;
        if (TOPK) {
          const uint32_t key = sortable_key(x);
          wi = topk_weight(key, tk_tau, tk_tw);
          wj = topk_weight(key, __shfl_sync(0xffffffffu, my_tau, j), __shfl_sync(0xffffffffu, my_tw, j));
        }
        const float g_ij = same ? (diag ? 0.f : cn_i * ptx::rcp_approx(e + neg_i)) : cs_i * e * wi;
        const float g_ji = same ? (diag ? 0.f : cnj * ptx::rcp_approx(e2 + negj)) : csj * e2 * wj;
        gv[j] = (!valid || lj == -2) ? 0.f : (g_ij + g_ji);
      }
    }
    // this thread's 32 columns = half of the G tile's 128-byte row: 4 chunks of 16 B, 128B-swizzled by row (the previous
    // tile's wgmma 2 has retired: it was waited for before this tile began)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int chunk = half * 4 + q;
      uint4 val = make_uint4(pack_bf16x2(gv[8 * q], gv[8 * q + 1]), pack_bf16x2(gv[8 * q + 2], gv[8 * q + 3]),
                             pack_bf16x2(gv[8 * q + 4], gv[8 * q + 5]), pack_bf16x2(gv[8 * q + 6], gv[8 * q + 7]));
      *reinterpret_cast<uint4*>(g_row + ((chunk ^ (r_in & 7)) << 4)) = val;
    }
    ptx::fence_proxy_async();                     // generic-proxy stores -> visible to the tensor core (async proxy)
    ptx::bar_sync(2 + g, 128);                    // G rows of the warpgroup complete; staging buffer free again
    // ---- wgmma 2: dA += G . C  (A operand: G, K-major, K = column j; B operand: the contrast tile read MN-major:
    // N = feature d (4 chunks of 64 at C_KB_BYTES), K = j (16 rows = 2 KB per step)) ----
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BNB / 16; ++k) {
      const uint64_t dg = ptx::make_desc_kmajor_sw128(g_base + k * 32);
      const uint64_t dc = ptx::make_desc_mnmajor_sw128(c_stage + k * 2048, C_KB_BYTES, 1024);
      ptx::wgmma_m64n256k16<1>(dacc, dg, dc, 1u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operands(dacc);
    if (lane == 0) ptx::mbar_arrive(&sm.c_empty[stage]);
  }
  // ---- dA of the warpgroup's rows -> global partial of this split (fragment layout, 8-byte stores) ----
  const int fr = 16 * (t >> 5) + ((t & 31) >> 2), fc = 2 * (t & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* dst = dpartials + ((int64_t)split * a.a_pad + row0 + g * 64 + fr + 8 * h) * DDIM + fc;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(dacc[4 * i + 2 * h], dacc[4 * i + 2 * h + 1]);
  }
}

// anchors fp32 -> bf16 rows (optional) and the per-row stabiliser m2 = |bf16(a)| * cbound * log2(e)/T
__global__ void k_tc_prep(const float* __restrict__ anchors, __nv_bfloat16* __restrict__ out_bf16,
                          const __nv_bfloat16* __restrict__ in_bf16, int a_rows, int a_pad, float cbound, float k1,
                          float* __restrict__ row_m2, float* __restrict__ partials, int64_t n_slot_rows) {
  // (a) partial slots that no CTA will write must read as "nothing seen": m = -inf, sums = 0
  if (partials != nullptr) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slot_rows; i += (int64_t)gridDim.x * blockDim.x) {
      partials[i] = -CUDART_INF_F;
#pragma unroll
      for (int k = 1; k < 5; ++k) partials[k * n_slot_rows + i] = 0.f;
    }
  }
  // (b) bf16 anchor rows (optional) and the per-row stabiliser
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= a_pad) return;
  float ss = 0.f;
  for (int d = lane; d < DDIM; d += 32) {
    __nv_bfloat16 h;
    if (out_bf16) {
      h = __float2bfloat16(r < a_rows ? anchors[(int64_t)r * DDIM + d] : 0.f);
      out_bf16[(int64_t)r * DDIM + d] = h;
    } else {
      h = in_bf16[(int64_t)r * DDIM + d];
    }
    const float f = __bfloat162float(h);
    ss += f * f;
  }
  ss = warp_sum(ss);
  if (lane == 0) row_m2[r] = sqrtf(ss) * cbound * k1 * 1.0001f;
}

// first column of every label for a sorted label array: start[L] = first n with ccls[n] >= L
__global__ void k_cls_bounds_init(int32_t* __restrict__ start, int n_cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= PCL_MAX_CLASSES) start[i] = n_cols;
}
__global__ void k_cls_bounds(const int32_t* __restrict__ ccls, int n_cols, int32_t* __restrict__ start) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_cols) return;
  const int cur = min(max(ccls[n], 0), PCL_MAX_CLASSES);
  const int prev = n == 0 ? -1 : min(max(ccls[n - 1], 0), PCL_MAX_CLASSES);
  for (int L = prev + 1; L <= cur; ++L) start[L] = n;
}

__global__ void k_to_bf16(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t n_real, int64_t n_total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16(i < n_real ? src[i] : 0.f);
}

}  // namespace tc
}  // namespace pcl

using namespace pcl;

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_tmapEncodeTiled)p;
  }
  return fn;
}

// Whether the calling thread has a current driver context (cuCtxGetCurrent; unknown -> false).
typedef CUresult (*PFN_ctxGetCurrent)(void**);
static bool has_current_context() {
  static PFN_ctxGetCurrent fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    const bool ok = cudaGetDriverEntryPoint("cuCtxGetCurrent", &p, cudaEnableDefault, &q) == cudaSuccess &&
                    q == cudaDriverEntryPointSuccess;
    return ok ? (PFN_ctxGetCurrent)p : (PFN_ctxGetCurrent) nullptr;
  }();
  void* ctx = nullptr;
  return fn != nullptr && fn(&ctx) == CUDA_SUCCESS && ctx != nullptr;
}

// Encoding a tensor map costs ~2 us of host time and the step re-uses the same few (pointer, shape, box) keys every
// call, so a small read-mostly cache keeps them (a tensor map only describes addresses/shapes: no lifetime coupling).
struct TmapKey { const void* base; uint64_t cols; uint64_t rows; uint32_t box_rows; };
struct TmapEntry { TmapKey k; CUtensorMap m; bool used; };
static TmapEntry g_tmaps[16];
static unsigned g_tmap_next = 0;
static std::mutex g_tmap_mu;

int pcl::tc_make_tmap(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows) {
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    for (auto& e : g_tmaps)
      if (e.used && e.k.base == base && e.k.cols == cols && e.k.rows == rows && e.k.box_rows == box_rows) {
        *m = e.m;
        return PCL_OK;
      }
  }
  PFN_tmapEncodeTiled enc = get_encode();
  if (!enc) { pcl::set_error_text("cuTensorMapEncodeTiled entry point not found"); return PCL_ERR_CUDA; }
  // cuTensorMapEncodeTiled is a DRIVER call: it needs a context current on THIS thread.  A thread that has not made a
  // runtime call yet (PyTorch's autograd worker on its first backward) has none -> CUDA_ERROR_INVALID_CONTEXT (201), seen
  // in tools/dist_bank_check.py.  cudaFree(0) binds the primary context.  Only then: during a stream capture (a thread
  // that is capturing has a context) cudaFree is a prohibited call and would invalidate the capture.
  if (!has_current_context()) (void)cudaFree(nullptr);
  cuuint64_t gdim[2] = {(cuuint64_t)cols, rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)tc::BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[256];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed (CUresult %d): base %p rows %llu box_rows %u", (int)r, base,
             (unsigned long long)rows, box_rows);
    pcl::set_error_text(msg);
    return PCL_ERR_CUDA;
  }
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  TmapEntry& e = g_tmaps[g_tmap_next++ % 16];
  e.k = TmapKey{base, cols, rows, box_rows};
  e.m = *m;
  e.used = true;
  return PCL_OK;
}

struct TcPlan {
  tc::TcArgs a;
  SweepArgs sw;         // for the shared combine / finalize kernels
  int row_tiles, grid_persistent, splits_bwd;
};

int pcl::num_sms() {
  static int cache[64] = {0};     // per device (a process may drive several GPUs)
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return 132; }   // sizing on a host without a device
  int& n = cache[dev & 63];
  if (n == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) n = v;
    else { (void)cudaGetLastError(); return 132; }
  }
  return n;
}

static int make_tc_plan(const pcl_tc_desc* d, TcPlan* p) {
  if (!d || !d->anchor_cls || d->a_rows <= 0) return PCL_ERR_ARG;
  if (d->D != tc::DDIM) return PCL_ERR_UNSUPPORTED;
  if (!(d->temperature > 0.f) || !(d->base_temperature > 0.f)) return PCL_ERR_ARG;
  memset(p, 0, sizeof(*p));
  tc::TcArgs& a = p->a;
  a.acls = d->anchor_cls; a.diag = d->diag_col; a.plan = d->plan; a.ccls = nullptr;
  a.a_rows = d->a_rows; a.mode = d->mode;
  p->row_tiles = ceil_div(d->a_rows, tc::BM);
  a.a_pad = p->row_tiles * tc::BM;
  int tail = 0;
  if (d->mode == 0) {
    // self-contrast: the columns are the anchors, which the engine keeps grouped by class (any grouping order makes
    // "first label == last label" a valid uniformity test for a 32-column chunk)
    a.n_cols = d->a_rows; a.sorted = d->sorted ? 1 : 0; a.K = 0; a.R = 1;
  } else if (d->mode == 1) {
    if (d->bank_K < 1 || d->bank_R < 1) return PCL_ERR_ARG;
    a.K = d->bank_K; a.R = d->bank_R; a.n_cols = (int64_t)(d->bank_K - 1) * d->bank_R; a.sorted = 1; tail = d->bank_R;
    if (d->bank_R < 2) return PCL_ERR_ARG;                      // (segment + pixel queue: R = 2M >= 2)
    tc::make_div((uint32_t)d->bank_R, &a.r_mul, &a.r_sh);
  } else if (d->mode == 2) {
    if (!d->contrast_cls || d->n_cols <= 0) return PCL_ERR_ARG;
    a.ccls = d->contrast_cls; a.n_cols = d->n_cols; a.sorted = d->sorted ? 1 : 0; a.K = 0; a.R = 1;
  } else {
    return PCL_ERR_ARG;
  }
  a.k1 = tc::LOG2E / d->temperature;
  a.tail_count = tail;
  const int sms = num_sms();
  const int col_tiles = (int)ceil_div64(a.n_cols > 0 ? a.n_cols : 1, tc::BN);
  int splits = sms / p->row_tiles;
  if (splits < 1) splits = 1;
  if (splits > col_tiles) splits = col_tiles;
  a.splits = splits;
  // persistent NEG sweep: G CTAs walk contiguous ranges of the row_tiles x col_tiles pair list
  const long long P = (long long)p->row_tiles * col_tiles;
  p->grid_persistent = (int)(P < sms ? P : sms);
  a.neg_grid = p->grid_persistent;
  long long slots_neg = d->plan ? (long long)p->grid_persistent                            // live A unknown on the host
                                : tc::neg_slot_bound(p->row_tiles, col_tiles, p->grid_persistent);
  if (slots_neg > p->grid_persistent) slots_neg = p->grid_persistent;
  if (slots_neg > col_tiles) slots_neg = col_tiles;
  if (slots_neg < 1) slots_neg = 1;
  a.slots = (int)(slots_neg > splits ? slots_neg : splits);
  // backward sweeps BNB-column tiles on a 2-D grid
  const int col_tiles_b = (int)ceil_div64(a.n_cols > 0 ? a.n_cols : 1, tc::BNB);
  int sb = sms / p->row_tiles;
  if (sb < 1) sb = 1;
  if (sb > col_tiles_b) sb = col_tiles_b;
  p->splits_bwd = sb;
  SweepArgs& s = p->sw;
  s.acls = d->anchor_cls; s.diag = d->diag_col; s.plan = d->plan;
  s.a_rows = d->a_rows; s.D = tc::DDIM; s.mode = d->mode;
  s.n_cols = a.n_cols; s.tail_count = tail;
  s.inv_T = 1.f / d->temperature; s.T_over_bT = d->temperature / d->base_temperature;
  s.nan_safe = d->nan_safe; s.row_tiles = p->row_tiles; s.splits = a.slots; s.a_pad = a.a_pad; s.col_tiles = col_tiles;
  s.pos_splits = a.splits;                 // the POS sweep runs on the 2-D grid: only its `splits` slots are written
  return PCL_OK;
}

extern "C" int pcl_tc_sizes(const pcl_tc_desc* d, pcl_sweep_sizes_t* out) {
  pcl_tc_desc tmp = *d;
  static const int32_t dummy = 0;
  tmp.anchor_cls = &dummy;
  if (tmp.mode == 2) tmp.contrast_cls = &dummy;
  TcPlan p;
  int st = make_tc_plan(&tmp, &p);
  if (st != PCL_OK || !out) return st != PCL_OK ? st : PCL_ERR_ARG;
  out->n_real_cols = p.a.n_cols;
  out->row_tiles = p.row_tiles;
  out->splits = p.a.slots;
  out->partial_f32 = (int64_t)p.a.slots * p.a.a_pad;
  out->rowstat_f32 = d->a_rows;
  out->dpartial_f32 = (int64_t)p.splits_bwd * p.a.a_pad * tc::DDIM;
  return PCL_OK;
}

extern "C" int pcl_to_bf16(const float* src, void* dst, int64_t n_real, int64_t n_total, void* stream) {
  PCL_REQUIRE(src && dst && n_total >= n_real && n_real >= 0);
  tc::k_to_bf16<<<num_sms() * 8, 256, 0, (cudaStream_t)stream>>>(src, (__nv_bfloat16*)dst, n_real, n_total);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

int pcl::tc_query(const pcl_tc_desc* d, int64_t* n_slot_rows, float* m2_scale) {
  TcPlan p;
  int st = make_tc_plan(d, &p);
  if (st != PCL_OK) return st;
  *n_slot_rows = (int64_t)p.a.slots * p.a.a_pad;
  const float cbound = d->contrast_norm_bound > 0.f ? d->contrast_norm_bound : 1.0f;
  *m2_scale = cbound * p.a.k1 * 1.0001f;
  return PCL_OK;
}

// The contrast operand of a descriptor as a tensor map of box_rows-row boxes: the anchors themselves in self-contrast
// mode, else the bf16 contrast rows (as many as allocated, or the real columns).
static int contrast_tmap(CUtensorMap* m, const pcl_tc_desc* d, const tc::TcArgs& a, uint32_t box_rows) {
  if (d->mode == 0) return tc_make_tmap(m, d->anchors_bf16, tc::DDIM, (uint64_t)a.a_pad, box_rows);
  return tc_make_tmap(m, d->contrast_bf16, tc::DDIM,
                      (uint64_t)(d->contrast_rows_alloc > 0 ? d->contrast_rows_alloc : a.n_cols), box_rows);
}

// Set-up of the row-tile forward sweeps: with `prep`, the bf16 anchors (if fp32 given) and the row stabilisers row_m2
// (contrast norm bound `cbound`), and the partial slots initialised when `partials` is given; then the tensor maps of the
// anchor tiles and of the contrast tiles.
static int fwd_setup(const pcl_tc_desc* d, const tc::TcArgs& a, bool prep, float cbound, float* row_m2, float* partials,
                     cudaStream_t s, CUtensorMap* tmA, CUtensorMap* tmB) {
  if (prep) {
    tc::k_tc_prep<<<ceil_div(a.a_pad, 8), 256, 0, s>>>(d->anchors_f32, d->anchors_f32 ? (__nv_bfloat16*)d->anchors_bf16 : nullptr,
                                                       (const __nv_bfloat16*)d->anchors_bf16, d->a_rows, a.a_pad, cbound,
                                                       a.k1, row_m2, partials, (int64_t)a.slots * a.a_pad);
    PCL_LAUNCH_CHECK();
  }
  const int st = tc_make_tmap(tmA, d->anchors_bf16, tc::DDIM, (uint64_t)a.a_pad, tc::BM);
  return st != PCL_OK ? st : contrast_tmap(tmB, d, a, tc::BN);
}

extern "C" int pcl_infonce_tc_fwd(const pcl_tc_desc* d, float* row_m2, float* partials, float* rowstats, float* loss,
                                  void* stream) {
  return pcl::tc_fwd_ex(d, row_m2, partials, rowstats, loss, stream, false, nullptr);
}

int pcl::tc_fwd_ex(const pcl_tc_desc* d, float* row_m2, float* partials, float* rowstats, float* loss, void* stream,
                   bool skip_prep, unsigned long long* step_counter) {
  return tc_fwd_topk_ex(d, 0, nullptr, row_m2, partials, rowstats, loss, stream, skip_prep, step_counter);
}

extern "C" int64_t pcl_tc_topk_scratch_u32(const pcl_tc_desc* d) {
  if (!d || d->a_rows <= 0) return PCL_ERR_ARG;
  const int64_t a_pad = (int64_t)ceil_div(d->a_rows, tc::BM) * tc::BM;
  return a_pad * TK_BINS + 4 * (int64_t)d->a_rows;
}

extern "C" int pcl_infonce_tc_topk_fwd(const pcl_tc_desc* d, int32_t k, uint32_t* scratch, float* row_m2, float* partials,
                                       float* rowstats, float* loss, void* stream) {
  if (k < 1 || !scratch) return PCL_ERR_ARG;
  return pcl::tc_fwd_topk_ex(d, k, scratch, row_m2, partials, rowstats, loss, stream, false, nullptr);
}

// k == 0: all negatives (the reference).  k >= 1 (a10): the negative sum keeps the k hardest negatives of every anchor:
// three histogram sweeps over the logit keys (per-row bins in global memory, red.global from the epilogue) with the
// warp-per-row scans of pcl_topk.cuh in between, then the weighted negative sweep; POS and finalize as usual.
int pcl::tc_fwd_topk_ex(const pcl_tc_desc* d, int k, uint32_t* scratch, float* row_m2, float* partials, float* rowstats,
                        float* loss, void* stream, bool skip_prep, unsigned long long* step_counter) {
  TcPlan p;
  int st = make_tc_plan(d, &p);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(row_m2 && partials && rowstats && loss && d->anchors_bf16);
  if (d->mode != 0) PCL_REQUIRE(d->contrast_bf16);
  cudaStream_t s = (cudaStream_t)stream;
  tc::TcArgs& a = p.a;
  a.row_m2 = row_m2;
  // (the step path has the anchor selection kernel write row_m2 and initialise the partial slots: skip_prep)
  const float cbound = d->contrast_norm_bound > 0.f ? d->contrast_norm_bound : 1.0f;
  CUtensorMap tmA, tmB;
  st = fwd_setup(d, a, !skip_prep, cbound, row_m2, partials, s, &tmA, &tmB);
  if (st != PCL_OK) return st;
  if (d->mode == 2 && a.sorted) {
    int32_t* cls_start = reinterpret_cast<int32_t*>(row_m2 + a.a_pad);       // scratch tail: PCL_MAX_CLASSES + 1 ints
    tc::k_cls_bounds_init<<<2, 256, 0, s>>>(cls_start, (int)a.n_cols);
    PCL_LAUNCH_CHECK();
    tc::k_cls_bounds<<<(unsigned)ceil_div64(a.n_cols, 256), 256, 0, s>>>(d->contrast_cls, (int)a.n_cols, cls_start);
    PCL_LAUNCH_CHECK();
    a.cls_start = cls_start;
  }
  const size_t smem = sizeof(tc::SmemLayout) + 1024;
  PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_NEG>, smem);
  PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_POS>, smem);
  a.persistent = 1;
  if (k >= 1) {
    PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_H1>, smem);
    PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_H2>, smem);
    PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_H3>, smem);
    PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_NEGW>, smem);
    TopkArgs tk;
    tk.k = k;
    tk.hist = scratch;
    tk.sel = scratch + (int64_t)a.a_pad * TK_BINS;
    a.tk_hist = tk.hist;
    a.tk_sel = tk.sel;
    PCL_CUDA(cudaMemsetAsync(tk.hist, 0, (size_t)a.a_pad * TK_BINS * sizeof(uint32_t), s));
    const int scan_blocks = ceil_div(d->a_rows, 8);          // 8 warps (rows) per 256-thread block
    tc::k_tc_fwd<tc::TC_H1><<<p.grid_persistent, tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, partials, nullptr);
    PCL_LAUNCH_CHECK();
    k_topk_scan<1><<<scan_blocks, 256, 0, s>>>(p.sw, tk);
    PCL_LAUNCH_CHECK();
    tc::k_tc_fwd<tc::TC_H2><<<p.grid_persistent, tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, partials, nullptr);
    PCL_LAUNCH_CHECK();
    k_topk_scan<2><<<scan_blocks, 256, 0, s>>>(p.sw, tk);
    PCL_LAUNCH_CHECK();
    tc::k_tc_fwd<tc::TC_H3><<<p.grid_persistent, tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, partials, nullptr);
    PCL_LAUNCH_CHECK();
    k_topk_scan<3><<<scan_blocks, 256, 0, s>>>(p.sw, tk);
    PCL_LAUNCH_CHECK();
    tc::k_tc_fwd<tc::TC_NEGW><<<p.grid_persistent, tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, partials, nullptr);
  } else {
    tc::k_tc_fwd<tc::TC_NEG><<<p.grid_persistent, tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, partials, nullptr);
  }
  PCL_LAUNCH_CHECK();
  a.persistent = 0;
  if (d->neg_only) return PCL_OK;     // similarity + negative-sum sweep only (roofline measurement)
  // (the NEG partials are combined by the POS sweep's row prologue: no separate pass)
  if (d->mode == 1 && d->a_rows <= tc::PT_MAX_ROWS) {
    // small anchor sets against the bank: the transposed POS sweep (work list by class, every epilogue lane busy)
    CUtensorMap tmA64, tmC128;
    st = tc_make_tmap(&tmA64, d->anchors_bf16, tc::DDIM, (uint64_t)a.a_pad, tc::PT_NB);
    if (st != PCL_OK) return st;
    st = contrast_tmap(&tmC128, d, a, tc::PT_BM);
    if (st != PCL_OK) return st;
    const size_t smem_pt = sizeof(tc::SmemPosT) + 1024;
    PCL_SMEM_OPT_IN(tc::k_tc_pos_t, smem_pt);
    tc::k_tc_pos_t<<<num_sms(), tc::NUM_THREADS, smem_pt, s>>>(tmA64, tmC128, a, partials, rowstats);
  } else {
    tc::k_tc_fwd<tc::TC_POS><<<dim3(p.row_tiles, a.splits), tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, partials, rowstats);
  }
  PCL_LAUNCH_CHECK();
  k_finalize<<<1, 1024, 0, s>>>(p.sw, partials, rowstats, loss, step_counter);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

// Descriptor / pipeline self-test: raw similarity tiles S = A . C^T (fp32 accumulate of bf16 operands) to `dump`
// ((a_rows rounded up to 128) x (n_cols rounded up to 256) floats).
extern "C" int pcl_tc_dump_logits(const pcl_tc_desc* d, float* row_m2, float* dump, void* stream) {
  TcPlan p;
  int st = make_tc_plan(d, &p);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(row_m2 && dump && d->anchors_bf16);
  cudaStream_t s = (cudaStream_t)stream;
  tc::TcArgs& a = p.a;
  a.row_m2 = row_m2;
  CUtensorMap tmA, tmB;
  st = fwd_setup(d, a, true, 1.f, row_m2, nullptr, s, &tmA, &tmB);
  if (st != PCL_OK) return st;
  const size_t smem = sizeof(tc::SmemLayout) + 1024;
  PCL_SMEM_OPT_IN(tc::k_tc_fwd<tc::TC_DUMP>, smem);
  tc::k_tc_fwd<tc::TC_DUMP><<<dim3(p.row_tiles, a.splits), tc::NUM_THREADS, smem, s>>>(tmA, tmB, a, dump, nullptr);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_infonce_tc_bwd(const pcl_tc_desc* d, const float* row_m2, const float* rowstats, const float* grad_loss,
                                  float* dpartials, float* dA, void* stream) {
  return pcl::tc_bwd_ex(d, row_m2, rowstats, grad_loss, dpartials, dA, stream, nullptr, nullptr);
}

extern "C" int pcl_infonce_tc_topk_bwd(const pcl_tc_desc* d, int32_t k, const uint32_t* scratch, const float* row_m2,
                                       const float* rowstats, const float* grad_loss, float* dpartials, float* dA,
                                       void* stream) {
  if (k < 1 || !scratch) return PCL_ERR_ARG;
  return pcl::tc_bwd_ex(d, row_m2, rowstats, grad_loss, dpartials, dA, stream, nullptr, nullptr, scratch);
}

// dA == nullptr: leave the per-split partials for a fused consumer (splits_out / a_pad_out describe their layout)
int pcl::tc_bwd_ex(const pcl_tc_desc* d, const float* row_m2, const float* rowstats, const float* grad_loss,
                   float* dpartials, float* dA, void* stream, int* splits_out, int* a_pad_out, const uint32_t* topk_scratch) {
  TcPlan p;
  int st = make_tc_plan(d, &p);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(row_m2 && rowstats && dpartials && d->anchors_bf16);
  if (d->mode != 0) PCL_REQUIRE(d->contrast_bf16);
  cudaStream_t s = (cudaStream_t)stream;
  tc::TcBwdArgs ba;
  ba.t = p.a;
  ba.t.row_m2 = row_m2;
  if (topk_scratch != nullptr) ba.t.tk_sel = topk_scratch + (int64_t)ba.t.a_pad * TK_BINS;      // a10 selection of the forward
  ba.rowstats = rowstats;
  ba.rs_scale = d->temperature / d->base_temperature;
  ba.nan_safe = d->nan_safe;
  const int splits = p.splits_bwd;       // the backward sweeps BNB-column tiles on a 2-D grid
  ba.t.splits = splits;
  p.sw.splits = splits;
  CUtensorMap tmA, tmC;
  st = tc_make_tmap(&tmA, d->anchors_bf16, tc::DDIM, (uint64_t)ba.t.a_pad, tc::BM);
  if (st != PCL_OK) return st;
  st = contrast_tmap(&tmC, d, ba.t, tc::BNB);
  if (st != PCL_OK) return st;
  const size_t smem = sizeof(tc::SmemBwd) + 1024;
  PCL_SMEM_OPT_IN((tc::k_tc_bwd<false>), smem);
  PCL_SMEM_OPT_IN((tc::k_tc_bwd<true>), smem);
  dim3 grid(p.row_tiles, splits);
  if (ba.t.tk_sel != nullptr) tc::k_tc_bwd<true><<<grid, tc::NUM_THREADS, smem, s>>>(tmA, tmC, ba, dpartials);
  else                        tc::k_tc_bwd<false><<<grid, tc::NUM_THREADS, smem, s>>>(tmA, tmC, ba, dpartials);
  PCL_LAUNCH_CHECK();
  if (splits_out) *splits_out = splits;
  if (a_pad_out) *a_pad_out = ba.t.a_pad;
  if (dA == nullptr) return PCL_OK;
  const int64_t total = (int64_t)d->a_rows * tc::DDIM;
  k_reduce_dA<<<(unsigned)ceil_div64(total, 256), 256, 0, s>>>(p.sw, dpartials, grad_loss, dA);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}
