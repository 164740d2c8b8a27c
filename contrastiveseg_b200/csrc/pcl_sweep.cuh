// Row-statistic kernels shared by the exact (SIMT) and the tensor-core InfoNCE sweeps.
// Partials layout: partials[(k * splits + split) * a_pad + row], k = 0: stabiliser m (natural-log logit units),
// 1: sum over negatives of exp(l - m), 2: sum over positives of log-prob, 3: sum over positives of 1/(e+Neg),
// 4: number of positives.  Row statistics layout: rowstats[k * a_rows + row], k = m, neg, possum, s, npos, row_loss.
#pragma once
#include "pcl_common.cuh"
#include <math_constants.h>

namespace pcl {

struct SweepArgs {
  const float* anchors; const int32_t* acls; const int32_t* diag; const int32_t* plan;
  int a_rows, D, mode;
  const float* segq; const float* pixq; int K, M0, M1, R;
  const float* contrast; const int32_t* ccls;
  int64_t n_cols;          // upper bound of streamed columns (self mode: a_rows)
  int tail_count;          // analytic all-zero columns with label 0 (bank mode: R)
  float inv_T, T_over_bT;
  int nan_safe;
  int row_tiles, splits, a_pad, col_tiles;
  int pos_splits;          // live slots of the POS partial arrays (0 = same as splits)
};

__device__ __forceinline__ int live_rows(const SweepArgs& a) {
  int A = a.plan ? a.plan[PCL_PLAN_A] : a.a_rows;
  return A < a.a_rows ? A : a.a_rows;
}


// Combine the POS partials, add the zero-tail positives of class-0 anchors, row losses and the mean.
static __global__ void __launch_bounds__(1024)
k_finalize(SweepArgs a, const float* __restrict__ partials, float* __restrict__ rowstats, float* __restrict__ loss,
           unsigned long long* step_counter) {
  // captured sequences: the selection (an earlier kernel) has drawn this step's anchors from *step_counter; advance it
  if (step_counter != nullptr && threadIdx.x == 0) *step_counter += 1ull;
  __shared__ float s_red[1024];
  const int A = live_rows(a);
  float acc = 0.f;
  for (int r = threadIdx.x; r < a.a_rows; r += blockDim.x) {
    float ps = 0.f, s = 0.f, c = 0.f, rl = 0.f;
    if (r < A) {
      const int npos = a.pos_splits > 0 ? a.pos_splits : a.splits;
      for (int p = 0; p < npos; ++p) {                 // fixed summation order
        ps += partials[((int64_t)2 * a.splits + p) * a.a_pad + r];
        s += partials[((int64_t)3 * a.splits + p) * a.a_pad + r];
        c += partials[((int64_t)4 * a.splits + p) * a.a_pad + r];
      }
      if (a.tail_count > 0 && a.acls[r] == 0) {
        const float m = rowstats[r], neg = rowstats[a.a_rows + r];
        const float t = expf(-m) + neg;
        // the masked (i,i) entry can fall inside the zero tail when A > (K-1)*R (Q1)
        const int dg = a.diag ? a.diag[r] : -1;
        const float tc = (float)(a.tail_count - ((dg >= a.n_cols && dg < a.n_cols + a.tail_count) ? 1 : 0));
        ps += tc * (-m - logf(t));
        s += tc / t;
        c += tc;
      }
      rl = -a.T_over_bT * ps / c;
      if (a.nan_safe && !(c > 0.f)) rl = 0.f;
      acc += rl;
    }
    rowstats[2 * a.a_rows + r] = ps;
    rowstats[3 * a.a_rows + r] = s;
    rowstats[4 * a.a_rows + r] = c;
    rowstats[5 * a.a_rows + r] = rl;
  }
  s_red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = A > 0 ? s_red[0] / (float)A : 0.f;
}

static __global__ void k_reduce_dA(SweepArgs a, const float* __restrict__ dpartials, const float* __restrict__ grad_loss,
                            float* __restrict__ dA) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)a.a_rows * a.D;
  if (idx >= total) return;
  const int r = (int)(idx / a.D);
  const int A = live_rows(a);
  float v = 0.f;
  if (r < A) {
    for (int p = 0; p < a.splits; ++p) v += dpartials[((int64_t)p * a.a_pad) * a.D + idx];
    v *= a.inv_T * (grad_loss ? *grad_loss : 1.f);
  }
  dA[idx] = v;
}


}  // namespace pcl
