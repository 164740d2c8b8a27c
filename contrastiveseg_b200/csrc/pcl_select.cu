// Anchor selection and gather/scatter kernels (SURVEY §8 rows a3, a4 and the dense-gradient writer).
//
// Replaces lib/loss/loss_contrast.py:30-89 (_hard_anchor_sampling) and :131-142 without the per-(image,
// class) Python loop, its ~5 host syncs per pair, and the 268 MB permute+contiguous copy:
//   k_keys    one pass over labels/seg: nearest-neighbour label, argmax, 16-bit key per pixel, and a
//             histogram of keys per 1024-pixel chunk (HBM-bound: reads B*K*h*w*4 B of seg once)
//   k_plan    class filter, TC, V, hard/easy split, class-sorted row layout (one block, integer only)
//   k_select  one warp per anchor: rank -> pixel (chunk prefix search + in-chunk ordered scan), gather
//             of the pixel's D channels from NCHW, optional L2-normalise, fp32 + bf16 rows
//   k_zero_scatter, k_scatter_reduce, k_scatter   the dense-gradient writers (dense_grad picks one)
#include "pcl_common.cuh"
#include <math_constants.h>

namespace pcl {

__device__ __forceinline__ void plan_body(const pcl_geom& g, const int32_t* counts, int32_t* plan);   // below (k_plan)

// ------------------------------------------------------------------------------------------------
// k_keys
// ------------------------------------------------------------------------------------------------
template <typename TS>      // element type of seg (the argmax compares the values converted to fp32)
__global__ void __launch_bounds__(PCL_CHUNK, 2)
k_keys(pcl_geom g, int nchunk, float scale_h, float scale_w, const int64_t* __restrict__ labels,
       const TS* __restrict__ seg, const int64_t* __restrict__ predict, uint16_t* __restrict__ keys,
       int32_t* chunk_hist, int32_t* counts, int32_t* plan, unsigned int* done_ctr) {
  extern __shared__ int s_hist[];                 // 2K+1 bins
  unsigned int* dbg = done_ctr ? done_ctr - 4 : nullptr;       // the step's sync buffer (timeline, diagnostics)
  tl_begin(dbg, PCL_TL_KEYS);
  const int K = g.K, NK = 2 * K;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int HW = g.h * g.w;
  for (int i = threadIdx.x; i <= NK; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const int p = chunk * PCL_CHUNK + threadIdx.x;   // one pixel per thread: coalesced plane reads, K loads in flight
  if (p < HW) {
    const int py = p / g.w, px = p - py * g.w;
    const int sy = nearest_src(py, scale_h, g.Himg), sx = nearest_src(px, scale_w, g.Wimg);
    const int64_t lab = labels[(int64_t)b * g.Himg * g.Wimg + (int64_t)sy * g.Wimg + sx];
    int key = NK;
    // K <= 32 (every configuration of the reference): the class-plane loads do not wait for the label — the label load
    // and the first 16 planes are one DRAM round trip, the remaining planes a second (was: label, then one round trip
    // per group of 8 planes behind the label test; the scan is a chain of dependent round trips).  16 at a time: 1024 threads x 32 registers keeps two CTAs per SM.
    int pred32 = -1;
    if (seg != nullptr && K <= 32) {
      const TS* sp = seg + (int64_t)b * K * HW + p;
      float best = -CUDART_INF_F;
      pred32 = 0;
#pragma unroll
      for (int c0 = 0; c0 < 32; c0 += 16) {
        if (c0 < K) {
          // kept in the input type until the compare.  Under the 32-register cap of this launch bound every instantiation
          // spills a little (ptxas, bytes stored / loaded): fp32 36 / 112 as before; bf16 and fp16 40 / 104 (52 / 132
          // when converted at load time)
          TS v[16];
#pragma unroll
          for (int u = 0; u < 16; ++u) v[u] = (c0 + u < K) ? __ldg(sp + (int64_t)(c0 + u) * HW) : from_f32<TS>(-CUDART_INF_F);
#pragma unroll
          for (int u = 0; u < 16; ++u)
            if (to_f32(v[u]) > best) { best = to_f32(v[u]); pred32 = c0 + u; }    // first maximum wins, like torch.max
        }
      }
    }
    if (lab >= 0 && lab < K && lab != (int64_t)g.ignore_label) {
      int pred;
      if (seg != nullptr && K <= 32) {
        pred = pred32;
      } else if (seg != nullptr) {
        const TS* sp = seg + (int64_t)b * K * HW + p;
        float best = -CUDART_INF_F;
        pred = 0;
        for (int c0 = 0; c0 < K; c0 += 8) {
          float v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = (c0 + u < K) ? to_f32(__ldg(sp + (int64_t)(c0 + u) * HW)) : -CUDART_INF_F;
#pragma unroll
          for (int u = 0; u < 8; ++u)
            if (v[u] > best) { best = v[u]; pred = c0 + u; }       // first maximum wins, like torch.max
        }
      } else {
        const int64_t pv = predict[(int64_t)b * HW + p];
        pred = (pv >= 0 && pv < K) ? (int)pv : -1;
      }
      key = 2 * (int)lab + (pred == (int)lab ? 1 : 0);
    }
    keys[(int64_t)b * HW + p] = (uint16_t)key;
    atomicAdd(&s_hist[key], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NK; i += blockDim.x) {
    const int v = s_hist[i];
    chunk_hist[((int64_t)b * NK + i) * nchunk + chunk] = v;
    if (v && done_ctr == nullptr) atomicAdd(&counts[b * NK + i], v);     // integer totals: order-independent
  }
  if (done_ctr == nullptr) return;
  // ---- fused tail (step path): the LAST block to finish sums the per-chunk histograms into the totals (no atomics, no
  //      memset) and computes the sampling plan — saves the single-CTA k_plan launch and the counts memset ----
  __shared__ int s_last;
  tl_end(dbg, 5);                                  // (diagnostics: end of the scan part of the last-arriving block)
  // release: the block barrier orders every thread's writes before thread 0, whose device-scope fence is cumulative —
  // ONE fence per block instead of 1024 (the grid-barrier idiom); acquire on the other side the same way
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int total = gridDim.x * gridDim.y;
    __threadfence();
    s_last = (atomicAdd(done_ctr, 1u) == total - 1u) ? 1 : 0;
    __threadfence();
  }
  __syncthreads();
  if (!s_last) { tl_end(dbg, PCL_TL_KEYS); return; }
  // Totals: one warp per (image, key) row, one chunk per lane, FOUR rows per pass so that a warp has four loads in
  // flight (a row-at-a-time loop costs one L2 round trip per row).  The totals also stay in shared memory for the plan (its loops re-read them).
  __shared__ int s_counts[4096];
  const int rows = g.B * NK;
  const bool in_smem = rows <= 4096;
  {
    const int wid = threadIdx.x >> 5, ln = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int base = wid; base < rows; base += 4 * nw) {
      int t[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = base + q * nw;
        t[q] = 0;
        if (i < rows) {
          const int32_t* hrow = chunk_hist + (int64_t)i * nchunk;
          for (int ch = ln; ch < nchunk; ch += 32) t[q] += __ldcg(hrow + ch);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t[q] += __shfl_xor_sync(0xffffffffu, t[q], o);
        const int i = base + q * nw;
        if (ln == 0 && i < rows) { counts[i] = t[q]; if (in_smem) s_counts[i] = t[q]; }
      }
    }
  }
  if (threadIdx.x == 0) *done_ctr = 0u;           // re-armed for the next launch
  __syncthreads();
  tl_end(dbg, 6);                                  // (diagnostics: totals done)
  plan_body(g, in_smem ? s_counts : counts, plan);
  tl_end(dbg, PCL_TL_KEYS);
}

// ------------------------------------------------------------------------------------------------
// k_plan (single block)
// plan layout: [0..16) header, then 8 int32 per pair: img, cls, n_hard, n_easy, keep_hard, keep_easy,
//              sorted_base (first class-sorted row of the pair), reserved
// ------------------------------------------------------------------------------------------------
constexpr int PLAN_THREADS = 256;

// Executed by the first PLAN_THREADS threads of a block whose ALL threads call it (it contains block barriers).
// Exclusive prefix sum over the first PLAN_THREADS (= 8 full warps) threads of the block; every thread of the block must
// call it (block barriers inside).  Returns the exclusive prefix of v (0 for the other threads), *total = the sum.
__device__ __forceinline__ int plan_scan(int v, bool act, int* s_w, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
  if (act) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) s_w[warp] = incl;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int w = 0; w < PLAN_THREADS / 32; ++w) { const int t = s_w[w]; s_w[w] = run; run += t; }
    s_w[PLAN_THREADS / 32] = run;
  }
  __syncthreads();
  *total = s_w[PLAN_THREADS / 32];
  const int excl = act ? incl - v + s_w[warp] : 0;
  __syncthreads();                                     // s_w may be re-used by the next scan
  return excl;
}

// (no __restrict__ / read-only path on `counts`: the fused scan's last block writes the totals itself just before)
__device__ __forceinline__ void plan_body(const pcl_geom& g, const int32_t* counts, int32_t* plan) {
  __shared__ int s_w[PLAN_THREADS / 32 + 1];
  __shared__ int s_cls_cnt[PCL_MAX_CLASSES];
  __shared__ int s_cls_start[PCL_MAX_CLASSES];
  __shared__ int s_err;
  const int K = g.K, NK = 2 * K, B = g.B;
  const int tid = threadIdx.x;
  const bool act = tid < PLAN_THREADS;                 // the other threads of a larger block only take part in barriers
  if (tid == 0) s_err = 0;
  if (act) for (int c = tid; c < K; c += PLAN_THREADS) s_cls_cnt[c] = 0;
  __syncthreads();

  // 1. kept (image,class) pairs in (image asc, class asc) order: thread t owns entries [t*per, (t+1)*per)
  const int E = B * K;
  const int per = (E + PLAN_THREADS - 1) / PLAN_THREADS;
  const int e0 = act ? min(E, tid * per) : E, e1 = act ? min(E, e0 + per) : E;
  int local = 0;
  for (int e = e0; e < e1; ++e) {
    int b = e / K, c = e - b * K;
    int n = counts[b * NK + 2 * c] + counts[b * NK + 2 * c + 1];
    local += (n > g.max_views) ? 1 : 0;
  }
  int TC = 0;
  int t = plan_scan(local, act, s_w, &TC);
  const int V = TC > 0 ? min(g.max_samples / TC, g.max_views) : 0;
  int32_t* pairs = plan + PCL_PLAN_HEADER;
  int split_err = 0;
  for (int e = e0; e < e1; ++e) {
    int b = e / K, c = e - b * K;
    int nh = counts[b * NK + 2 * c], ne = counts[b * NK + 2 * c + 1];
    if (nh + ne > g.max_views) {
      int kh, ke;
      // loss_contrast.py:66-77   (num >= n_view / 2  <=>  2*num >= n_view)
      if (2 * nh >= V && 2 * ne >= V) { kh = V / 2; ke = V - kh; }
      else if (2 * nh >= V)           { ke = ne;    kh = V - ke; }
      else if (2 * ne >= V)           { kh = nh;    ke = V - kh; }
      else                            { kh = 0; ke = 0; split_err = 1; }
      int32_t* q = pairs + (int64_t)t * 8;
      q[0] = b; q[1] = c; q[2] = nh; q[3] = ne; q[4] = kh; q[5] = ke; q[6] = 0; q[7] = 0;
      atomicAdd(&s_cls_cnt[c], 1);
      ++t;
    }
  }
  if (split_err) atomicOr(&s_err, 1);
  __syncthreads();
  // 2. class-sorted start rows, rank order 1,2,...,K-1,0 (K <= 256 = PLAN_THREADS: one rank per thread)
  {
    const int rnk = tid;
    const int c = (rnk == K - 1) ? 0 : rnk + 1;
    const int v = (act && rnk < K) ? s_cls_cnt[c] : 0;
    int tot = 0;
    const int start = plan_scan(v, act, s_w, &tot);
    if (act && rnk < K) s_cls_start[c] = start;
  }
  if (tid == 0) {
    plan[PCL_PLAN_TC] = TC;
    plan[PCL_PLAN_V] = V;
    plan[PCL_PLAN_A] = TC * V;
    int f = s_err ? PCL_FLAG_SPLIT_ERROR : 0;
    if (TC == 0) f |= PCL_FLAG_NO_CLASS;
    if (TC > 0 && V == 0) f |= PCL_FLAG_ZERO_VIEWS;
    plan[PCL_PLAN_FLAGS] = f;
    plan[PCL_PLAN_NPAIR_MAX] = E;
    for (int i = PCL_PLAN_NPAIR_MAX + 1; i < PCL_PLAN_HEADER; ++i) plan[i] = 0;
  }
  __syncthreads();
  // 3. sorted base per pair: V * (class start + number of earlier images that kept the class)
  for (int p = act ? tid : TC; p < TC; p += PLAN_THREADS) {
    int32_t* q = pairs + (int64_t)p * 8;
    int b = q[0], c = q[1];
    int before = 0;
    for (int bb = 0; bb < b; ++bb) {
      int n = counts[bb * NK + 2 * c] + counts[bb * NK + 2 * c + 1];
      before += (n > g.max_views) ? 1 : 0;
    }
    q[6] = V * (s_cls_start[c] + before);
  }
}

__global__ void __launch_bounds__(PLAN_THREADS)
k_plan(pcl_geom g, int nchunk, const int32_t* __restrict__ counts, int32_t* __restrict__ plan) {
  plan_body(g, counts, plan);
}

// ------------------------------------------------------------------------------------------------
// k_select: one warp per anchor row
// ------------------------------------------------------------------------------------------------
template <typename T>       // element type of embed and grad_clear
__global__ void __launch_bounds__(256)
k_select(pcl_geom g, int nchunk, const T* __restrict__ embed, const uint16_t* __restrict__ keys,
         const int32_t* __restrict__ chunk_pref, const int32_t* __restrict__ plan,
         const int32_t* __restrict__ ranks, uint64_t seed, int normalize, int32_t* __restrict__ meta,
         float* __restrict__ anchors, __nv_bfloat16* __restrict__ anchors_bf16, float* __restrict__ inv_norm,
         float* __restrict__ norm_max, float* __restrict__ row_m2, float m2_scale, float* __restrict__ partials,
         int64_t n_slot_rows, const unsigned long long* __restrict__ seed_ctr, unsigned int* dbg,
         const int32_t* __restrict__ prev_rows, T* __restrict__ grad_clear) {
  tl_begin(dbg, PCL_TL_SELECT);
  struct TlEnd { unsigned int* d; __device__ ~TlEnd() { tl_end(d, PCL_TL_SELECT); } } tl_guard{dbg};
  // Sparse reset (persistent dense-gradient buffer of a captured step): instead of re-filling B*D*h*w zeros every step,
  // clear exactly the entries the PREVIOUS step scattered (prev_rows: [0] = A_prev, then pixel[ms], image[ms]); the
  // buffer is zero everywhere else by induction.  Runs before this step's scatter (stream order).
  if (prev_rows != nullptr) {
    const int ip = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int msp = g.max_samples;
    if (ip < min(prev_rows[0], msp)) {
      const int64_t HWp = (int64_t)g.h * g.w;
      T* dstp = grad_clear + (int64_t)prev_rows[1 + msp + ip] * g.D * HWp + prev_rows[1 + ip];
      for (int d = threadIdx.x & 31; d < g.D; d += 32) dstp[(int64_t)d * HWp] = from_f32<T>(0.f);
    }
  }
  // captured launch sequences: the per-step part of the seed lives in device memory (same formula as pcl_step_ranks)
  if (seed_ctr != nullptr) seed = seed * 0x9E3779B97F4A7C15ull + *seed_ctr + 1ull;
  // tensor-path fusion: initialise the partial-statistic slots (m = -inf, sums = 0) while we are here
  if (partials != nullptr) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_slot_rows; k += (int64_t)gridDim.x * blockDim.x) {
      partials[k] = -CUDART_INF_F;
#pragma unroll
      for (int q = 1; q < 5; ++q) partials[q * n_slot_rows + k] = 0.f;
    }
  }
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int TC = plan[PCL_PLAN_TC], V = plan[PCL_PLAN_V];
  const int D = g.D, ms = g.max_samples;
  if (i >= ms) {
    // padding rows of the bf16 copy (rounded up to 128 rows for the 128-row TMA boxes)
    if (anchors_bf16 != nullptr && i < ((ms + 127) / 128) * 128) {
      for (int d = lane; d < D; d += 32) anchors_bf16[(int64_t)i * D + d] = __float2bfloat16(0.f);
      if (row_m2 != nullptr && lane == 0) row_m2[i] = 0.f;
    }
    return;
  }
  if (V <= 0 || i >= TC * V) {
    // dead row (the class-sorted rows [0, A) are dense): zero it so padded tiles read zeros
    for (int d = lane; d < D; d += 32) {
      anchors[(int64_t)i * D + d] = 0.f;
      if (anchors_bf16 != nullptr) anchors_bf16[(int64_t)i * D + d] = __float2bfloat16(0.f);
    }
    if (lane == 0) {
      meta[i] = -1; meta[ms + i] = -1; meta[2 * ms + i] = -1; meta[3 * ms + i] = -1; inv_norm[i] = 0.f;
      if (row_m2 != nullptr) row_m2[i] = 0.f;
    }
    return;
  }
  const int t = i / V, v = i - t * V;
  const int32_t* q = plan + PCL_PLAN_HEADER + (int64_t)t * 8;
  const int b = q[0], c = q[1], nh = q[2], ne = q[3], kh = q[4], base = q[6];
  const int K = g.K, NK = 2 * K, HW = g.h * g.w;
  const bool easy = v >= kh;
  const int j = easy ? v - kh : v;
  const int n = easy ? ne : nh;
  const int key = 2 * c + (easy ? 1 : 0);
  int rank;
  if (ranks != nullptr) rank = ranks[(int64_t)t * V + v];
  else rank = (int)keyed_perm((uint32_t)j, (uint32_t)n, mix64(seed ^ ((uint64_t)(b * K + c) << 1 | (easy ? 1u : 0u))));
  if (rank < 0) rank = 0;
  if (rank >= n) rank = n - 1;               // defensive: malformed injected table

  // chunk that holds the rank-th pixel of this key: warp scan of the per-chunk histogram row
  const int32_t* hist = chunk_pref + ((int64_t)b * NK + key) * nchunk;
  int chunk = -1, local = 0, run = 0;
  for (int c0 = 0; c0 < nchunk && chunk < 0; c0 += 32) {
    const int ch = c0 + lane;
    const int cnt = ch < nchunk ? hist[ch] : 0;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    const int lo = run + incl - cnt;
    const unsigned m = __ballot_sync(0xffffffffu, cnt > 0 && rank >= lo && rank < lo + cnt);
    if (m) {
      const int src = __ffs(m) - 1;
      chunk = c0 + src;
      local = rank - __shfl_sync(0xffffffffu, lo, src);
    }
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (chunk < 0) return;                       // cannot happen for a consistent table

  // ordered scan of the chunk: lane L owns pixels [32L, 32L+32)
  const int p0 = chunk * PCL_CHUNK + lane * 32;
  const uint16_t* kb = keys + (int64_t)b * HW;
  // the lane's 32 keys (64 bytes) in four 16-byte loads when the row base allows it (HW % 8 == 0: always for the step's
  // geometries), kept in registers for both passes below
  uint16_t kv[32];
  if ((HW & 7) == 0 && p0 + 32 <= HW) {
    const uint4* k4 = reinterpret_cast<const uint4*>(kb + p0);
#pragma unroll
    for (int w4 = 0; w4 < 4; ++w4) {
      const uint4 x = __ldg(k4 + w4);
      const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) { kv[w4 * 8 + 2 * e] = (uint16_t)(xs[e] & 0xFFFFu); kv[w4 * 8 + 2 * e + 1] = (uint16_t)(xs[e] >> 16); }
    }
  } else {
#pragma unroll
    for (int u = 0; u < 32; ++u) kv[u] = (p0 + u < HW) ? kb[p0 + u] : (uint16_t)0xFFFFu;
  }
  int cnt = 0;
#pragma unroll
  for (int u = 0; u < 32; ++u) cnt += (p0 + u < HW && kv[u] == (uint16_t)key) ? 1 : 0;
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  const int excl = incl - cnt;
  int pix = -1;
  if (local >= excl && local < incl) {
    int need = local - excl;
#pragma unroll
    for (int u = 0; u < 32; ++u) {
      if (p0 + u < HW && kv[u] == (uint16_t)key) {
        if (need == 0 && pix < 0) pix = p0 + u;
        --need;
      }
    }
  }
  unsigned owner = __ballot_sync(0xffffffffu, pix >= 0);
  if (!owner) return;
  pix = __shfl_sync(0xffffffffu, pix, __ffs(owner) - 1);

  // gather the D channels of (b, pix)
  const int s = base + v;
  const T* src = embed + (int64_t)b * D * HW + pix;
  float* dst = anchors + (int64_t)s * D;
  float ss = 0.f;
  for (int d = lane; d < D; d += 32) {
    float x = to_f32(src[(int64_t)d * HW]);
    ss += x * x;
    dst[d] = x;
  }
  ss = warp_sum(ss);
  const float nrm = sqrtf(ss);
  const float inv = normalize ? 1.f / fmaxf(nrm, 1e-12f) : 1.f;
  float ss16 = 0.f;                           // squared norm of the bf16-rounded row (tensor-path stabiliser)
  for (int d = lane; d < D; d += 32) {
    float y = dst[d] * inv;
    if (normalize) dst[d] = y;
    if (anchors_bf16 != nullptr) {
      const __nv_bfloat16 hb = __float2bfloat16(y);
      anchors_bf16[(int64_t)s * D + d] = hb;
      const float f = __bfloat162float(hb);
      ss16 += f * f;
    }
  }
  if (row_m2 != nullptr) {
    ss16 = warp_sum(ss16);
    if (lane == 0) row_m2[s] = sqrtf(ss16) * m2_scale;
  }
  if (lane == 0) {
    meta[s] = pix;
    meta[ms + s] = b;
    meta[2 * ms + s] = c;
    meta[3 * ms + s] = v * TC + t;
    inv_norm[s] = inv;
    if (norm_max != nullptr) atomicMax(reinterpret_cast<int*>(norm_max), __float_as_int(nrm * inv));
  }
}

// ------------------------------------------------------------------------------------------------
// k_scatter: dA rows -> dense NCHW gradient (buffer is zeroed by a memset first)
// ------------------------------------------------------------------------------------------------
template <typename T>       // element type of grad: the fp32 value is rounded once
__global__ void __launch_bounds__(256)
k_scatter(pcl_geom g, const int32_t* __restrict__ plan, const int32_t* __restrict__ meta,
          const float* __restrict__ dA, const float* __restrict__ anchors, const float* __restrict__ inv_norm,
          int normalize, T* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int A = plan[PCL_PLAN_A];
  if (s >= A) return;
  const int ms = g.max_samples, D = g.D;
  const int64_t HW = (int64_t)g.h * g.w;
  const int pix = meta[s], b = meta[ms + s];
  const float* ga = dA + (int64_t)s * D;
  float dot = 0.f, inv = 1.f;
  if (normalize) {
    const float* y = anchors + (int64_t)s * D;
    for (int d = lane; d < D; d += 32) dot += y[d] * ga[d];
    dot = warp_sum(dot);
    inv = inv_norm[s];
  }
  T* dst = grad + (int64_t)b * D * HW + pix;
  for (int d = lane; d < D; d += 32) {
    float v = ga[d];
    if (normalize) v = (v - anchors[(int64_t)s * D + d] * dot) * inv;
    dst[(int64_t)d * HW] = from_f32<T>(v);
  }
}

// ------------------------------------------------------------------------------------------------
// Anchor rows of the dense gradient: the (A, D) matrix dA, or (step path: the matrix is never written) the backward
// sweep's per-split partial rows, value = scale * sum_p dpartials[p][s][d].
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float split_sum(const float* dpartials, int splits, int a_pad, int D, int s, int d) {
  float v = 0.f;
  for (int p = 0; p < splits; ++p) v += __ldg(dpartials + ((int64_t)p * a_pad + s) * D + d);     // fixed order
  return v;
}

struct DaRows {                      // dA's value as it is: a zero-gradient row may hold -0, which 0.f + x would lose
  const float* dA;
  __device__ float scale() const { return 1.f; }
  __device__ float at(int s, int d, int D, float) const { return __ldg(dA + (int64_t)s * D + d); }
};

struct SplitRows {
  const float* dpartials;
  int splits, a_pad;
  float inv_T;
  const float* grad_scale;           // device scalar (captured steps rescale it between replays), null = 1
  __device__ float scale() const { return inv_T * (grad_scale ? __ldg(grad_scale) : 1.f); }
  __device__ float at(int s, int d, int D, float scale) const { return split_sum(dpartials, splits, a_pad, D, s, d) * scale; }
};

// Zero-fills one (image, channel) plane of HW elements, with 16-byte stores when the plane allows them.
template <typename T>
__device__ __forceinline__ void zero_plane(T* dst, int64_t HW) {
  constexpr int E = 16 / sizeof(T);                // elements per 16-byte store
  if (HW % E == 0) {
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (int64_t i = threadIdx.x; i < HW / E; i += blockDim.x) d4[i] = z;
  } else {
    for (int64_t i = threadIdx.x; i < HW; i += blockDim.x) dst[i] = from_f32<T>(0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// k_zero_scatter: the dense gradient in ONE pass — each CTA owns one (image, channel) plane of h*w floats, zero-fills
// it with 16-byte stores and then drops in the gradient entries of the anchors sampled from that image.
// HBM-bound: writes B*D*h*w*4 bytes once (the floor of the backward: autograd needs the dense tensor).
// ------------------------------------------------------------------------------------------------
template <typename T, typename Src>
__global__ void __launch_bounds__(256)
k_zero_scatter(pcl_geom g, const int32_t* __restrict__ plan, const int32_t* __restrict__ meta, Src src,
               T* __restrict__ grad) {
  const int plane = blockIdx.x;
  const int D = g.D, ms = g.max_samples;
  const int b = plane / D, d = plane - b * D;
  const int64_t HW = (int64_t)g.h * g.w;
  T* dst = grad + (int64_t)plane * HW;
  zero_plane(dst, HW);
  __syncthreads();
  const int A = min(plan[PCL_PLAN_A], ms);
  const float scale = src.scale();
  for (int s = threadIdx.x; s < A; s += blockDim.x)
    if (meta[ms + s] == b) dst[meta[s]] = from_f32<T>(src.at(s, d, D, scale));
}

// Scatter of the A gradient rows into an ALREADY zero-filled dense gradient, with the fixed-order sum of the per-split
// (per-column-tile) partial rows folded in: one block per anchor row.  Also advances the step counter of a captured
// sequence (last kernel of the step).
template <typename T>
__global__ void __launch_bounds__(256)
k_scatter_reduce(pcl_geom g, const int32_t* __restrict__ plan, const int32_t* __restrict__ meta, SplitRows src,
                 int split_cols, T* __restrict__ grad, unsigned long long* step_counter, unsigned int* dbg,
                 int32_t* __restrict__ prev_rows) {
  // one BLOCK per anchor row, one thread per channel: the sum over the splits (up to 18 for the bank sweeps) is a chain
  // of dependent adds per element, so the parallelism has to come from the elements (a warp per row leaves few warps
  // per SM)
  tl_begin(dbg, PCL_TL_SCATTER);
  struct TlEnd { unsigned int* d; __device__ ~TlEnd() { tl_end(d, PCL_TL_SCATTER); } } tl_guard{dbg};
  if (step_counter != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *step_counter += 1ull;
  const int s = blockIdx.x;
  const int A = min(plan[PCL_PLAN_A], g.max_samples);
  if (prev_rows != nullptr && s == 0 && threadIdx.x == 0) prev_rows[0] = A;           // what the next step has to clear
  if (s >= A) return;
  // partial p covers the contrast columns [p * split_cols, (p+1) * split_cols): only the live ones were written
  if (split_cols > 0) src.splits = min(src.splits, (A + split_cols - 1) / split_cols);
  const int ms = g.max_samples, D = g.D;
  const int64_t HW = (int64_t)g.h * g.w;
  const int pix = meta[s], b = meta[ms + s];
  if (prev_rows != nullptr && threadIdx.x == 0) { prev_rows[1 + s] = pix; prev_rows[1 + ms + s] = b; }
  const float scale = src.scale();
  // Whole 32-byte sectors: a store of 4 (2) bytes into a sector the fill left dirty in L2, or evicted, costs a
  // read-modify-write of the sector; the zeros around the anchor's pixel are written with it (measured on H100 after a
  // 268 MB fill: 1024 x 256 scattered 4-byte stores 26 us, the same stores as whole sectors 17 us).  Another sampled
  // pixel of the same image may share the sector: the anchor of lowest index writes the sector with every value in it,
  // the others write nothing.  Needs sector-aligned planes (the buffer is zero before the scatter: all callers).
  constexpr int E = 32 / (int)sizeof(T);            // elements per 32-byte sector
  if (HW % E == 0 && ((uintptr_t)grad & 31) == 0) {
    __shared__ int s_own[E];                        // anchor whose pixel is element j of the sector, -1 = zero
    __shared__ int s_skip;
    const int sec = pix - pix % E;
    if (threadIdx.x < E) s_own[threadIdx.x] = -1;
    if (threadIdx.x == 0) s_skip = 0;
    __syncthreads();
    for (int r = threadIdx.x; r < A; r += blockDim.x) {
      const int q = meta[r];
      if (meta[ms + r] == b && q - q % E == sec) {  // r == s included; sampled pixels are distinct
        s_own[q - sec] = r;
        if (r < s) s_skip = 1;
      }
    }
    __syncthreads();
    if (s_skip) return;
    const int j = threadIdx.x % E, own = s_own[j];
    T* row = grad + (int64_t)b * D * HW + sec + j;
    for (int d = threadIdx.x / E; d < D; d += blockDim.x / E)
      row[(int64_t)d * HW] = from_f32<T>(own >= 0 ? src.at(own, d, D, scale) : 0.f);   // +0 where no anchor, whatever the scale
    return;
  }
  T* dst = grad + (int64_t)b * D * HW + pix;
  for (int d = threadIdx.x; d < D; d += blockDim.x) dst[(int64_t)d * HW] = from_f32<T>(src.at(s, d, D, scale));
}

// Zero-fill with 16-byte stores (the dense gradient: B*D*h*w*4 bytes, the HBM floor of the step), four independent
// stores per iteration.
__device__ __forceinline__ void fill_loop(uint4* __restrict__ p, uint64_t n16) {
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) { p[i] = z; p[i + stride] = z; p[i + 2 * stride] = z; p[i + 3 * stride] = z; }
  for (; i < n16; i += stride) p[i] = z;
}

// Small footprint (256 threads, no shared memory) so that its CTAs share the SMs with the latency-bound kernels of the
// step.
__global__ void __launch_bounds__(256)
k_fill_zero(uint4* __restrict__ p, uint64_t n16, unsigned int* dbg) {
  tl_begin(dbg, PCL_TL_FILL);
  fill_loop(p, n16);
  tl_end(dbg, PCL_TL_FILL);
}

// The same fill as a few CTAs that OWN their SM (1024 threads + a dynamic shared-memory request no other kernel of the
// step fits next to): a CTA of another kernel that shares an SM with fill warps queues its loads, shuffles and shared-
// memory accesses behind the fill's stores and becomes the straggler of its kernel.
__global__ void __launch_bounds__(1024, 1)
k_fill_zero_excl(uint4* __restrict__ p, uint64_t n16, unsigned int* dbg) {
  extern __shared__ uint8_t fill_smem_unused[];
  tl_begin(dbg, PCL_TL_FILL);
  fill_loop(p, n16);
  tl_end(dbg, PCL_TL_FILL);
}

}  // namespace pcl

using namespace pcl;

extern "C" int pcl_fill_zero(void* ptr, uint64_t bytes, void* stream) { return pcl::fill_zero(ptr, bytes, stream, nullptr, 0); }

// reserve_sms: SMs to leave free of fill CTAs for a kernel that runs next to the fill (the fused InfoNCE kernel)
int pcl::fill_zero(void* ptr, uint64_t bytes, void* stream, unsigned int* dbg, int reserve_sms) {
  PCL_REQUIRE(ptr && (bytes & 15) == 0 && ((uintptr_t)ptr & 15) == 0);
  if (bytes == 0) return PCL_OK;
  const uint64_t n16 = bytes >> 4;
  const int sms = num_sms(), free_sms = sms - reserve_sms;
  // reserve_sms > 0: the caller runs a kernel of `reserve_sms` big CTAs next to the fill -> fill CTAs that own their SMs
  // (k_fill_zero_excl), on all SMs but the reserved ones
  if (reserve_sms > 0 && free_sms >= sms / 2 && free_sms >= 1) {
    // ALL of the SM's shared memory (227 KB + the 1 KB the system reserves per CTA): no other CTA fits next to it
    const size_t smem = 232448;
    PCL_SMEM_OPT_IN(k_fill_zero_excl, smem);
    k_fill_zero_excl<<<(unsigned)free_sms, 1024, smem, (cudaStream_t)stream>>>((uint4*)ptr, n16, dbg);
    PCL_LAUNCH_CHECK();
    return PCL_OK;
  }
  // One CTA per SM, on at least half of them: the fill is a long-running branch that shares the SMs with the
  // latency-bound kernels of the step; a few resident warps per SM saturate the HBM write path (stores do not wait),
  // more would only crowd the others out (the fill time does not depend on 1, 2, 4 or 8 CTAs per SM).
  uint64_t blocks = (n16 + 255) / 256;
  if (blocks > (uint64_t)max(free_sms, sms / 2)) blocks = max(free_sms, sms / 2);
  k_fill_zero<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((uint4*)ptr, n16, dbg);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

int pcl::dense_grad(const pcl_geom* g, const int32_t* plan, const int32_t* anchor_meta, const grad_rows& r, bool zeroed,
                    void* grad_embed, int grad_dtype, void* stream, unsigned int* dbg, unsigned long long* step_counter,
                    int32_t* prev_rows) {
  if (!g || !plan || !anchor_meta || !grad_embed || !dtype_ok(grad_dtype)) return PCL_ERR_ARG;
  const bool partial_rows = r.dpartials != nullptr;
  if (partial_rows ? r.splits < 1 || r.normalize : !r.dA || (r.normalize && (!r.anchors_f32 || !r.inv_norm)))
    return PCL_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  const SplitRows sp{r.dpartials, r.splits, r.a_pad, r.inv_T, r.grad_scale};
  if (!zeroed && !r.normalize) {                 // one pass: zero-fill and scatter per (image, channel) plane
    const unsigned planes = (unsigned)(g->B * g->D);
    PCL_DT_SWITCH(grad_dtype, T,
      if (!partial_rows) k_zero_scatter<T, DaRows><<<planes, 256, 0, s>>>(*g, plan, anchor_meta, DaRows{r.dA}, (T*)grad_embed);
      else               k_zero_scatter<T, SplitRows><<<planes, 256, 0, s>>>(*g, plan, anchor_meta, sp, (T*)grad_embed);)
  } else if (partial_rows) {                     // into the zeroed buffer, one block per anchor row
    PCL_DT_SWITCH(grad_dtype, T,
      k_scatter_reduce<T><<<g->max_samples, g->D <= 128 ? 128 : 256, 0, s>>>(
          *g, plan, anchor_meta, sp, r.split_cols, (T*)grad_embed, step_counter, dbg, prev_rows);)
  } else {                                       // the normalise projection, or a zeroed buffer: one warp per anchor row
    if (!zeroed) PCL_CUDA(cudaMemsetAsync(grad_embed, 0, (size_t)g->B * g->D * g->h * g->w * dtype_size(grad_dtype), s));
    const int warps = 8;
    PCL_DT_SWITCH(grad_dtype, T,
      k_scatter<T><<<ceil_div(g->max_samples, warps), warps * 32, 0, s>>>(*g, plan, anchor_meta, r.dA, r.anchors_f32,
                                                                         r.inv_norm, r.normalize, (T*)grad_embed);)
  }
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

// ==================================================================================================
// C ABI
// ==================================================================================================
static int check_geom(const pcl_geom* g) {
  if (!g) return PCL_ERR_ARG;
  if (g->B <= 0 || g->D <= 0 || g->h <= 0 || g->w <= 0 || g->Himg <= 0 || g->Wimg <= 0) return PCL_ERR_ARG;
  // the widths the sweeps take: refused here, before the scan and the selection run, not after them
  if (g->D % 32 != 0 || g->D > 256) return PCL_ERR_UNSUPPORTED;
  if (g->K <= 0 || g->K > PCL_MAX_CLASSES) return PCL_ERR_ARG;
  if (g->max_samples <= 0 || g->max_views <= 0) return PCL_ERR_ARG;
  if ((int64_t)g->B * g->K > (1 << 20)) return PCL_ERR_ARG;
  return PCL_OK;
}

extern "C" int pcl_select_sizes(const pcl_geom* g, pcl_select_sizes_t* out) {
  int st = check_geom(g);
  if (st != PCL_OK || !out) return PCL_ERR_ARG;
  const int64_t HW = (int64_t)g->h * g->w;
  out->nchunk = (int32_t)ceil_div64(HW, PCL_CHUNK);
  out->max_pairs = g->B * g->K;
  out->keys_u16 = (int64_t)g->B * HW;
  out->chunk_pref_i32 = (int64_t)g->B * 2 * g->K * out->nchunk;
  out->counts_i32 = (int64_t)g->B * 2 * g->K;
  out->plan_i32 = PCL_PLAN_HEADER + 8 * (int64_t)out->max_pairs;
  out->anchor_meta_i32 = 4 * (int64_t)g->max_samples;
  return PCL_OK;
}

extern "C" int pcl_class_stats(const pcl_geom* g, const int64_t* labels, const float* seg, const int64_t* predict,
                               uint16_t* keys, int32_t* chunk_pref, int32_t* counts, void* stream) {
  return pcl::class_stats(g, labels, seg, predict, keys, chunk_pref, counts, nullptr, nullptr, stream, PCL_DT_F32);
}

// done_ctr (one zeroed word; the step path): scan + totals + plan in ONE launch, the last block to finish runs the plan.
// Without it the totals are atomics into the zeroed counts and the plan is left to k_plan.
int pcl::class_stats(const pcl_geom* g, const int64_t* labels, const void* seg, const int64_t* predict, uint16_t* keys,
                     int32_t* chunk_pref, int32_t* counts, int32_t* plan, unsigned int* done_ctr, void* stream,
                     int seg_dtype) {
  int st = check_geom(g);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(labels && keys && chunk_pref && counts && (plan || !done_ctr) && (seg || predict) && dtype_ok(seg_dtype));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t HW = (int64_t)g->h * g->w;
  const int nchunk = (int)ceil_div64(HW, PCL_CHUNK);
  const float scale_h = (float)g->Himg / (float)g->h, scale_w = (float)g->Wimg / (float)g->w;
  if (!done_ctr) PCL_CUDA(cudaMemsetAsync(counts, 0, (size_t)g->B * 2 * g->K * sizeof(int32_t), s));
  dim3 grid(nchunk, g->B);
  size_t smem = (2 * g->K + 1) * sizeof(int);
  PCL_DT_SWITCH(seg_dtype, T,
    k_keys<T><<<grid, PCL_CHUNK, smem, s>>>(*g, nchunk, scale_h, scale_w, labels, (const T*)seg, predict, keys, chunk_pref,
                                            counts, plan, done_ctr);)
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_plan_anchors(const pcl_geom* g, const int32_t* counts, int32_t* plan, void* stream) {
  int st = check_geom(g);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(counts && plan);
  cudaStream_t s = (cudaStream_t)stream;
  const int nchunk = (int)ceil_div64((int64_t)g->h * g->w, PCL_CHUNK);
  k_plan<<<1, PLAN_THREADS, 0, s>>>(*g, nchunk, counts, plan);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

int pcl::select_gather(const select_args& a, void* stream) {
  const pcl_geom* g = a.g;
  int st = check_geom(g);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(a.embed && a.keys && a.chunk_pref && a.plan && a.anchor_meta && a.anchors_f32 && a.inv_norm &&
              dtype_ok(a.embed_dtype));
  cudaStream_t s = (cudaStream_t)stream;
  const int ms = g->max_samples;
  const int nchunk = (int)ceil_div64((int64_t)g->h * g->w, PCL_CHUNK);
  if (a.norm_max) PCL_CUDA(cudaMemsetAsync(a.norm_max, 0, sizeof(float), s));     // optional output
  const int warps = 8;
  // rows in [A, max_samples) are zero-filled by the kernel itself (no separate memsets); the bf16 copy is padded to
  // a multiple of 128 rows: cover those too
  const int rows = a.anchors_bf16 ? ceil_div(ms, 128) * 128 : ms;
  PCL_DT_SWITCH(a.embed_dtype, T,
    k_select<T><<<ceil_div(rows, warps), warps * 32, 0, s>>>(*g, nchunk, (const T*)a.embed, a.keys, a.chunk_pref, a.plan,
                                                             a.ranks, a.seed, a.normalize, a.anchor_meta, a.anchors_f32,
                                                             (__nv_bfloat16*)a.anchors_bf16, a.inv_norm, a.norm_max,
                                                             a.row_m2, a.m2_scale, a.partials, a.n_slot_rows, a.seed_ctr,
                                                             a.dbg, a.prev_rows, (T*)a.grad_clear);)
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_select_gather(const pcl_geom* g, const float* embed, const uint16_t* keys,
                                 const int32_t* chunk_pref, const int32_t* plan, const int32_t* ranks,
                                 uint64_t seed, int normalize, int32_t* anchor_meta, float* anchors_f32,
                                 void* anchors_bf16, float* inv_norm, float* norm_max, void* stream) {
  pcl::select_args a = {};
  a.g = g; a.embed = embed; a.embed_dtype = PCL_DT_F32; a.keys = keys; a.chunk_pref = chunk_pref; a.plan = plan;
  a.ranks = ranks; a.seed = seed; a.normalize = normalize; a.anchor_meta = anchor_meta; a.anchors_f32 = anchors_f32;
  a.anchors_bf16 = anchors_bf16; a.inv_norm = inv_norm; a.norm_max = norm_max;
  return pcl::select_gather(a, stream);
}

extern "C" int pcl_scatter_grad(const pcl_geom* g, const int32_t* plan, const int32_t* anchor_meta, const float* dA,
                                const float* anchors_f32, const float* inv_norm, int normalize, float* grad_embed,
                                void* stream) {
  int st = check_geom(g);
  if (st != PCL_OK) return st;
  pcl::grad_rows r = {};
  r.dA = dA; r.anchors_f32 = anchors_f32; r.inv_norm = inv_norm; r.normalize = normalize;
  return pcl::dense_grad(g, plan, anchor_meta, r, false, grad_embed, PCL_DT_F32, stream);
}
