// a10 (SURVEY §8): pieces of the per-anchor top-k hard-negative selection shared by the exact fp32 sweep
// (pcl_infonce_simt.cu) and the tensor-core sweep (pcl_infonce_tc.cu): the order-preserving key, the selection state,
// the radix-level scan.
#pragma once
#include "pcl_common.cuh"
#include "pcl_sweep.cuh"

namespace pcl {

constexpr int TK_BINS = 2048;
constexpr uint32_t TK_ALL = 0xFFFFFFFFu;      // selection state: the row keeps every negative
constexpr uint32_t KEY_ZERO = 0x80000000u;    // sortable key of +0.0f (the zero-tail logit)

struct TopkArgs {
  int k;
  uint32_t* hist;      // [a_pad][TK_BINS] per-row bins of the current radix level (zero between levels)
  uint32_t* sel;       // [4][a_rows]: key prefix -> tau key | remaining rank -> tie weight (float bits) | G | E
};

// order-preserving map fp32 -> uint32 (-0 folded into +0)
__device__ __forceinline__ uint32_t sortable_key(float l) {
  uint32_t u = __float_as_uint(l);
  if ((u << 1) == 0u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float topk_weight(uint32_t key, uint32_t tau, float tie_w) {
  return key > tau ? 1.f : (key == tau ? tie_w : 0.f);
}

// One warp per anchor row: walk the bins of the current radix level from the largest key down to the bin that holds
// the row's remaining rank, narrow the key prefix, and clear the bins for the next level.
template <int LEVEL>
__global__ void __launch_bounds__(256) k_topk_scan(SweepArgs a, TopkArgs tk) {
  const int r = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= a.a_rows) return;
  const int A = live_rows(a);
  uint32_t* sel_key = tk.sel;
  uint32_t* sel_rem = tk.sel + a.a_rows;
  uint32_t* sel_G = tk.sel + 2 * (int64_t)a.a_rows;
  uint32_t* sel_E = tk.sel + 3 * (int64_t)a.a_rows;
  constexpr uint32_t FULL = 0xffffffffu;
  const uint32_t one_bits = __float_as_uint(1.f);

  if (r >= A) {                                // dead row: neutral selection
    if (lane == 0) {
      if (LEVEL == 1) { sel_key[r] = TK_ALL; sel_rem[r] = 0u; sel_G[r] = 0u; sel_E[r] = 0u; }
      if (LEVEL == 3) { sel_key[r] = 0u; sel_rem[r] = one_bits; }
    }
    return;
  }
  const uint32_t prefix = LEVEL == 1 ? 0u : sel_key[r];
  if (LEVEL > 1 && prefix == TK_ALL) {         // decided at level 1: every negative is kept
    if (LEVEL == 3 && lane == 0) { sel_key[r] = 0u; sel_rem[r] = one_bits; }
    return;
  }
  const uint32_t need = LEVEL == 1 ? (uint32_t)tk.k : sel_rem[r];
  constexpr int NB = LEVEL == 3 ? 1024 : 2048;
  constexpr int CB = NB / 32;
  uint32_t* h = tk.hist + (int64_t)r * TK_BINS;

  // analytic zero tail (Q3): tail_count columns with logit +0, negatives of every anchor whose class is not 0
  int tail_bin = -1;
  if (a.tail_count > 0 && a.acls[r] != 0) {
    if (LEVEL == 1) tail_bin = (int)(KEY_ZERO >> 21);
    if (LEVEL == 2 && prefix == (KEY_ZERO >> 21)) tail_bin = (int)((KEY_ZERO >> 10) & 0x7FFu);
    if (LEVEL == 3 && prefix == (KEY_ZERO >> 10)) tail_bin = (int)(KEY_ZERO & 0x3FFu);
  }
  const uint32_t tail = (uint32_t)a.tail_count;

  // lane L owns bins [NB-(L+1)*CB, NB-L*CB): lane 0 holds the largest keys
  const int hi = NB - lane * CB, lo = hi - CB;
  uint32_t s = 0;
  for (int b = lo; b < hi; ++b) s += h[b] + (b == tail_bin ? tail : 0u);
  uint32_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t v = __shfl_up_sync(FULL, incl, o);
    if (lane >= o) incl += v;
  }
  const uint32_t above = incl - s;
  const uint32_t total = __shfl_sync(FULL, incl, 31);

  const bool mine = above < need && need <= above + s;
  const unsigned bal = __ballot_sync(FULL, mine);
  const bool keep_all = (LEVEL == 1 && total <= need) || bal == 0u;
  uint32_t f_bin = 0, f_rem = 0, f_cnt = 0;
  if (!keep_all && mine) {
    uint32_t cum = above;
    for (int b = hi - 1; b >= lo; --b) {
      const uint32_t c = h[b] + (b == tail_bin ? tail : 0u);
      if (cum + c >= need) { f_bin = (uint32_t)b; f_rem = need - cum; f_cnt = c; break; }
      cum += c;
    }
  }
  const int src = keep_all ? 0 : (__ffs(bal) - 1);
  f_bin = __shfl_sync(FULL, f_bin, src);
  f_rem = __shfl_sync(FULL, f_rem, src);
  f_cnt = __shfl_sync(FULL, f_cnt, src);
  __syncwarp();
  for (int b = lo; b < hi; ++b) h[b] = 0u;     // clean bins for the next level / the next call

  if (lane == 0) {
    if (keep_all) {
      if (LEVEL == 1) { sel_G[r] = total; sel_E[r] = 0u; }     // G = number of negatives of the row
      if (LEVEL == 3) { sel_key[r] = 0u; sel_rem[r] = one_bits; }
      else { sel_key[r] = TK_ALL; sel_rem[r] = 0u; }
    } else if (LEVEL == 1) {
      sel_key[r] = f_bin; sel_rem[r] = f_rem;
    } else if (LEVEL == 2) {
      sel_key[r] = (prefix << 11) | f_bin; sel_rem[r] = f_rem;
    } else {
      sel_key[r] = (prefix << 10) | f_bin;                                 // tau key
      sel_rem[r] = __float_as_uint((float)f_rem / (float)f_cnt);           // weight of each of the E ties
      sel_G[r] = (uint32_t)tk.k - f_rem;                                   // negatives strictly above tau
      sel_E[r] = f_cnt;
    }
  }
}


}  // namespace pcl
