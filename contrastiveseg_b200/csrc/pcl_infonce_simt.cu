// Exact-fp32 InfoNCE sweep (SURVEY §8 rows a5, a6, a10) — SIMT tiles, no A x N temporaries.
//
// Replaces lib/loss/loss_contrast.py:91-128 and lib/loss/loss_contrast_mem.py:91-152 (the dense
// A x N matmul and ~12 dense A x N temporaries, and the 194.6 MB torch.cat + _sample_negative copies:
// the two queues are read in place, the all-zero tail of the flattened bank is handled analytically).
//
// Three sweeps over (row tile 64) x (column tile 64) logit tiles, column range split across CTAs:
//   NEG  per-row running (max, sum of exp over negatives)            -> partial (m, neg) per split
//   POS  per-row sum over positives of log-prob, of 1/(e+Neg), count -> partial per split
//   BWD  recompute logits, form the gradient tile G (closed form), dA += G . C
// Row statistics are combined in fixed split order, so results are bit-reproducible.
// This is the exact path (fp32 FMA); the bf16 wgmma path lives in pcl_infonce_tc.cu.
//
// a10, per-anchor top-k hard negatives (an extension the reference does not have: loss_contrast.py:116-117 sums ALL
// negatives; semantics in oracle/ref_port.py: infonce_topk and include/pcl.h).  The A x N logits are never stored: an
// exact 3-level radix select (11 + 11 + 10 bits) on the order-preserving integer image of the fp32 logit — the
// histogram sweeps H1..H3 with per-row bins in global memory, each followed by a warp-per-row scan (pcl_topk.cuh) —
// then the weighted NEG sweep (NEGW), the stock POS sweep and finalize; the backward is the weighted BWD sweep (BWDW).
// The logit of an (anchor, column) pair is the same float in all five top-k sweeps (same FMA order, explicit round of
// the 1/T product); the exact sweeps keep the 1/T product contractible into the following subtraction.
#include "pcl_common.cuh"
#include "pcl_sweep.cuh"
#include "pcl_simt_tile.cuh"
#include "pcl_topk.cuh"

namespace pcl {

enum { MODE_NEG = 0, MODE_POS = 1, MODE_BWD = 2,
       MODE_H1 = 3, MODE_H2 = 4, MODE_H3 = 5, MODE_NEGW = 6, MODE_BWDW = 7 };      // top-k: histograms, weighted NEG / BWD

// tk: read by the top-k modes only (last parameter: the other modes keep their parameter offsets)
template <int MODE>
__global__ void __launch_bounds__(SWEEP_THREADS, 1)
k_sweep(SweepArgs a, float* __restrict__ partials, const float* __restrict__ rowstats, float* __restrict__ dpartials,
        TopkArgs tk) {
  constexpr bool TOPK = MODE >= MODE_H1;
  constexpr bool HIST = MODE >= MODE_H1 && MODE <= MODE_H3;
  constexpr bool NEG = MODE == MODE_NEG || MODE == MODE_NEGW;
  constexpr bool BWD = MODE == MODE_BWD || MODE == MODE_BWDW;
  extern __shared__ __align__(16) float smem[];
  const int D = a.D;
  float* As_t = smem;                         // [D][LDT]
  float* Ct = As_t + D * LDT;                 // [D][LDT]
  float* Gs = Ct + D * LDT;                   // [TM][LDT]   (BWD only)
  float* s_extra = Gs + (BWD ? TM * LDT : 0);
  const float** s_ptr = reinterpret_cast<const float**>(s_extra);                  // [64]
  int* s_rcls = reinterpret_cast<int*>(s_ptr + 64);                                // [64]
  int* s_rdiag = s_rcls + 64;                                                      // [64]
  int* s_clab = s_rdiag + 64;                                                      // [64] (-2 = invalid column)
  float* s_rm = reinterpret_cast<float*>(s_clab + 64);                             // [64]
  float* s_rneg = s_rm + 64;
  float* s_rs = s_rneg + 64;
  float* s_rc = s_rs + 64;
  float* s_cm = s_rc + 64;                                                         // column stats (self BWD)
  float* s_cneg = s_cm + 64;
  float* s_cs = s_cneg + 64;
  float* s_cc = s_cs + 64;
  uint32_t* s_rtau = reinterpret_cast<uint32_t*>(s_cc + 64);                       // top-k row: key prefix / tau key
  float* s_rw = reinterpret_cast<float*>(s_rtau + 64);                             // top-k row: weight of the ties
  uint32_t* s_ctau = reinterpret_cast<uint32_t*>(s_rw + 64);                       // column as anchor (self BWDW)
  float* s_cw = reinterpret_cast<float*>(s_ctau + 64);

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int rt = blockIdx.x, split = blockIdx.y;
  const int A = live_rows(a);
  const int row0 = rt * TM;
  if (row0 >= A) return;
  const int64_t ncols = a.mode == 0 ? (int64_t)A : a.n_cols;
  const float rs_scale = a.T_over_bT / (float)A;

  // ---- row tile: pointers, labels, stats ----
  if (tid < 64) {
    int r = row0 + tid;
    bool ok = r < A;
    s_ptr[tid] = ok ? a.anchors + (int64_t)r * D : nullptr;
    s_rcls[tid] = ok ? a.acls[r] : -1;
    s_rdiag[tid] = ok ? (a.mode == 0 ? r : (a.diag ? a.diag[r] : -1)) : -1;
    if (TOPK) {
      s_rtau[tid] = (ok && MODE != MODE_H1) ? tk.sel[r] : TK_ALL;
      s_rw[tid] = (ok && (MODE == MODE_NEGW || MODE == MODE_BWDW)) ? __uint_as_float(tk.sel[a.a_rows + r]) : 0.f;
    }
    if (MODE == MODE_POS || BWD) {
      const float* st = rowstats;
      s_rm[tid] = ok ? st[r] : 0.f;
      s_rneg[tid] = ok ? st[a.a_rows + r] : 1.f;
      if (BWD) {
        s_rs[tid] = ok ? st[3 * a.a_rows + r] : 0.f;
        float np = ok ? st[4 * a.a_rows + r] : 1.f;
        float c = rs_scale / np;
        if (a.nan_safe && !(np > 0.f)) c = 0.f;
        s_rc[tid] = ok ? c : 0.f;
      }
    }
  }
  __syncthreads();
  load_tile_T(As_t, s_ptr, D);

  // ---- column tile range of this CTA ----
  int t_lo = 0, t_hi = (int)((ncols + TN - 1) / TN);
  if (MODE == MODE_POS && a.mode == 1) {
    // rows are sorted by class rank 1..K-1,0; real positive columns exist for ranks <= K-2
    int last = (A - 1 - row0 < TM - 1) ? (A - 1 - row0) : (TM - 1);
    int rk_f = class_rank(s_rcls[0], a.K), rk_l = class_rank(s_rcls[last], a.K);
    if (rk_l > a.K - 2) rk_l = a.K - 2;
    if (rk_f > rk_l) { t_lo = 0; t_hi = 0; }
    else {
      t_lo = (int)(((int64_t)rk_f * a.R) / TN);
      t_hi = (int)((((int64_t)(rk_l + 1) * a.R) + TN - 1) / TN);
    }
  }
  const int span = t_hi - t_lo;
  const int per = (span + a.splits - 1) / a.splits;
  const int my_lo = t_lo + split * per;
  const int my_hi = min(t_hi, my_lo + per);

  float run_m[4], run_a[4], run_b[4];          // NEG: (max, sum) ; POS: (possum, s, count in run_m)
#pragma unroll
  for (int i = 0; i < 4; ++i) { run_m[i] = NEG ? -CUDART_INF_F : 0.f; run_a[i] = 0.f; run_b[i] = 0.f; }
  float dacc[4][QMAX];
  if (BWD) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int q = 0; q < QMAX; ++q) dacc[i][q] = 0.f;
  }
  const int nq = D / 16;

  for (int ct = my_lo; ct < my_hi; ++ct) {
    __syncthreads();                          // previous tile fully consumed (Ct, Gs, column arrays)
    if (tid < 64) {
      int64_t n = (int64_t)ct * TN + tid;
      int lab = -2;
      const float* p = nullptr;
      if (n < ncols) p = col_row(a, n, lab);
      s_ptr[tid] = p;
      s_clab[tid] = lab;
      if (BWD && a.mode == 0) {
        bool ok = n < ncols;
        s_cm[tid] = ok ? rowstats[n] : 0.f;
        s_cneg[tid] = ok ? rowstats[a.a_rows + n] : 1.f;
        s_cs[tid] = ok ? rowstats[3 * a.a_rows + n] : 0.f;
        float np = ok ? rowstats[4 * a.a_rows + n] : 1.f;
        float c = rs_scale / np;
        if (a.nan_safe && !(np > 0.f)) c = 0.f;
        s_cc[tid] = ok ? c : 0.f;
        if (TOPK) {
          s_ctau[tid] = ok ? tk.sel[n] : TK_ALL;
          s_cw[tid] = ok ? __uint_as_float(tk.sel[a.a_rows + n]) : 0.f;
        }
      }
    }
    __syncthreads();
    load_tile_T(Ct, s_ptr, D);
    __syncthreads();

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 8
    for (int k = 0; k < D; ++k) {
      float4 av = *reinterpret_cast<const float4*>(As_t + k * LDT + ty * 4);
      float4 bv = *reinterpret_cast<const float4*>(Ct + k * LDT + tx * 4);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }

    const int64_t col_base = (int64_t)ct * TN + tx * 4;
    if (HIST) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = ty * 4 + i;
        const int rcls = s_rcls[r];
        const uint32_t prefix = s_rtau[r];
        uint32_t* hrow = tk.hist + (int64_t)(row0 + r) * TK_BINS;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int lab = s_clab[tx * 4 + j];
          if (lab != -2 && rcls >= 0 && lab != rcls) {
            const uint32_t key = sortable_key(__fmul_rn(acc[i][j], a.inv_T));
            if (MODE == MODE_H1) {
              atomicAdd(hrow + (key >> 21), 1u);
            } else if (MODE == MODE_H2) {
              if ((key >> 21) == prefix) atomicAdd(hrow + ((key >> 10) & 0x7FFu), 1u);
            } else {
              if ((key >> 10) == prefix) atomicAdd(hrow + (key & 0x3FFu), 1u);
            }
          }
        }
      }
    } else if (MODE == MODE_NEGW) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = ty * 4 + i;
        const int rcls = s_rcls[r];
        const uint32_t tau = s_rtau[r];
        const float tw = s_rw[r];
        float lv[4];
        float tmax = -CUDART_INF_F;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          lv[j] = __fmul_rn(acc[i][j], a.inv_T);
          if (s_clab[tx * 4 + j] != -2) tmax = fmaxf(tmax, lv[j]);
        }
        if (tmax > run_m[i]) {
          run_a[i] = (run_m[i] == -CUDART_INF_F) ? 0.f : run_a[i] * expf(run_m[i] - tmax);
          run_m[i] = tmax;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int lab = s_clab[tx * 4 + j];
          if (lab != -2 && lab != rcls) {
            const float w = topk_weight(sortable_key(lv[j]), tau, tw);
            if (w > 0.f) run_a[i] += w * expf(lv[j] - run_m[i]);
          }
        }
      }
    } else if (MODE == MODE_NEG) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int rcls = s_rcls[ty * 4 + i];
        float tmax = -CUDART_INF_F;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (s_clab[tx * 4 + j] != -2) tmax = fmaxf(tmax, acc[i][j] * a.inv_T);
        if (tmax > run_m[i]) {
          run_a[i] = (run_m[i] == -CUDART_INF_F) ? 0.f : run_a[i] * expf(run_m[i] - tmax);
          run_m[i] = tmax;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int lab = s_clab[tx * 4 + j];
          if (lab != -2 && lab != rcls) run_a[i] += expf(acc[i][j] * a.inv_T - run_m[i]);
        }
      }
    } else if (MODE == MODE_POS) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = ty * 4 + i;
        const int rcls = s_rcls[r], rdiag = s_rdiag[r];
        const float m = s_rm[r], neg = s_rneg[r];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int lab = s_clab[tx * 4 + j];
          if (lab == rcls && rcls >= 0 && (col_base + j) != (int64_t)rdiag) {
            float lm = acc[i][j] * a.inv_T - m;
            float t = expf(lm) + neg;
            run_a[i] += lm - logf(t);
            run_b[i] += 1.f / t;
            run_m[i] += 1.f;
          }
        }
      }
    } else {
      // gradient tile G (closed form, SURVEY appendix A; BWDW: the selection weight on the negatives)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = ty * 4 + i;
        const int rcls = s_rcls[r], rdiag = s_rdiag[r];
        const float m = s_rm[r], neg = s_rneg[r], S = s_rs[r], c = s_rc[r];
        const uint32_t tau = TOPK ? s_rtau[r] : 0u;
        const float tw = TOPK ? s_rw[r] : 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cj = tx * 4 + j;
          const int lab = s_clab[cj];
          float gval = 0.f;
          if (lab != -2 && rcls >= 0) {
            const float l = TOPK ? __fmul_rn(acc[i][j], a.inv_T) : acc[i][j] * a.inv_T;
            const uint32_t key = TOPK ? sortable_key(l) : 0u;
            const float e = expf(l - m);
            if (lab == rcls) {
              if ((col_base + j) != (int64_t)rdiag) gval = -c * (1.f - e / (e + neg));
            } else {
              gval = TOPK ? c * e * S * topk_weight(key, tau, tw) : c * e * S;
            }
            if (a.mode == 0) {               // + G_ji: the column is an anchor too (self-contrast); l_ji == l_ij bitwise
              const float e2 = expf(l - s_cm[cj]);
              if (lab == rcls) {
                if ((col_base + j) != (int64_t)rdiag) gval += -s_cc[cj] * (1.f - e2 / (e2 + s_cneg[cj]));
              } else {
                gval += TOPK ? s_cc[cj] * e2 * s_cs[cj] * topk_weight(key, s_ctau[cj], s_cw[cj]) : s_cc[cj] * e2 * s_cs[cj];
              }
            }
          }
          Gs[r * LDT + cj] = gval;
        }
      }
      __syncthreads();
      // dA[r][d] += sum_j G[r][j] * C[j][d],  C[j][d] = Ct[d*LDT + j]
#pragma unroll 4
      for (int j4 = 0; j4 < TN; j4 += 4) {
        float4 gv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) gv[i] = *reinterpret_cast<const float4*>(Gs + (ty * 4 + i) * LDT + j4);
#pragma unroll
        for (int q = 0; q < QMAX; ++q) {
          if (q < nq) {
            float4 cv = *reinterpret_cast<const float4*>(Ct + (tx + 16 * q) * LDT + j4);
#pragma unroll
            for (int i = 0; i < 4; ++i)
              dacc[i][q] += gv[i].x * cv.x + gv[i].y * cv.y + gv[i].z * cv.z + gv[i].w * cv.w;
          }
        }
      }
    }
  }

  // ---- write partials (the histogram modes write none) ----
  if (NEG) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float m = run_m[i], n = run_a[i];
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        float om = __shfl_xor_sync(0xffffffffu, m, o), on = __shfl_xor_sync(0xffffffffu, n, o);
        float nm = fmaxf(m, om);
        float s0 = (m == -CUDART_INF_F) ? 0.f : n * expf(m - nm);
        float s1 = (om == -CUDART_INF_F) ? 0.f : on * expf(om - nm);
        n = s0 + s1; m = nm;
      }
      if (tx == 0) {
        int r = row0 + ty * 4 + i;
        partials[((int64_t)0 * a.splits + split) * a.a_pad + r] = m;
        partials[((int64_t)1 * a.splits + split) * a.a_pad + r] = n;
      }
    }
  } else if (MODE == MODE_POS) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float p = run_a[i], s = run_b[i], c = run_m[i];
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        p += __shfl_xor_sync(0xffffffffu, p, o);
        s += __shfl_xor_sync(0xffffffffu, s, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
      }
      if (tx == 0) {
        int r = row0 + ty * 4 + i;
        partials[((int64_t)2 * a.splits + split) * a.a_pad + r] = p;
        partials[((int64_t)3 * a.splits + split) * a.a_pad + r] = s;
        partials[((int64_t)4 * a.splits + split) * a.a_pad + r] = c;
      }
    }
  } else if (BWD) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int r = row0 + ty * 4 + i;
      float* dst = dpartials + ((int64_t)split * a.a_pad + r) * D;
#pragma unroll
      for (int q = 0; q < QMAX; ++q)
        if (q < nq) dst[tx + 16 * q] = dacc[i][q];
    }
  }
}

// Combine the NEG partials of all splits (fixed order) and add the analytic zero tail (Q3), with the selection weight of
// the tail under top-k (tk: read by k_combine_neg<true> only).
template <bool TOPK>
static __global__ void k_combine_neg(SweepArgs a, const float* __restrict__ partials, float* __restrict__ rowstats,
                                     TopkArgs tk) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int A = live_rows(a);
  if (r >= a.a_rows) return;
  if (r >= A) { rowstats[r] = 0.f; rowstats[a.a_rows + r] = 0.f; return; }
  float m = -CUDART_INF_F;
  for (int p = 0; p < a.splits; ++p) m = fmaxf(m, partials[((int64_t)0 * a.splits + p) * a.a_pad + r]);
  if (a.tail_count > 0) m = fmaxf(m, 0.f);
  float n = 0.f;
  for (int p = 0; p < a.splits; ++p) {
    float pm = partials[((int64_t)0 * a.splits + p) * a.a_pad + r];
    if (pm != -CUDART_INF_F) n += partials[((int64_t)1 * a.splits + p) * a.a_pad + r] * expf(pm - m);
  }
  if (a.tail_count > 0 && a.acls[r] != 0)
    n += TOPK ? topk_weight(KEY_ZERO, tk.sel[r], __uint_as_float(tk.sel[a.a_rows + r])) * (float)a.tail_count * expf(-m)
              : (float)a.tail_count * expf(-m);
  rowstats[r] = m;
  rowstats[a.a_rows + r] = n;
}

}  // namespace pcl

using namespace pcl;

int pcl::simt_make_args(const pcl_sweep_desc* d, SweepArgs* a) {
  if (!d || !d->anchors || !d->anchor_cls) return PCL_ERR_ARG;
  if (d->a_rows <= 0 || d->D <= 0) return PCL_ERR_ARG;
  if (d->D % 32 != 0 || d->D > 256) return PCL_ERR_UNSUPPORTED;
  if (!(d->temperature > 0.f) || !(d->base_temperature > 0.f)) return PCL_ERR_ARG;
  memset(a, 0, sizeof(*a));
  a->anchors = d->anchors; a->acls = d->anchor_cls; a->diag = d->diag_col; a->plan = d->plan;
  a->a_rows = d->a_rows; a->D = d->D; a->mode = d->mode;
  if (d->mode == 0) {
    a->n_cols = d->a_rows; a->tail_count = 0;
  } else if (d->mode == 1) {
    if (!d->segment_queue || d->bank_K < 1 || d->bank_M0 < 1 || d->bank_M1 < 0) return PCL_ERR_ARG;
    if (d->bank_M1 > 0 && !d->pixel_queue) return PCL_ERR_ARG;
    a->segq = d->segment_queue; a->pixq = d->pixel_queue; a->K = d->bank_K; a->M0 = d->bank_M0; a->M1 = d->bank_M1;
    a->R = d->bank_M0 + d->bank_M1;
    a->n_cols = (int64_t)(d->bank_K - 1) * a->R; a->tail_count = a->R;
  } else if (d->mode == 2) {
    if (!d->contrast || !d->contrast_cls || d->n_cols <= 0) return PCL_ERR_ARG;
    a->contrast = d->contrast; a->ccls = d->contrast_cls; a->n_cols = d->n_cols; a->tail_count = 0;
  } else {
    return PCL_ERR_ARG;
  }
  a->inv_T = 1.f / d->temperature;
  a->T_over_bT = d->temperature / d->base_temperature;
  a->nan_safe = d->nan_safe;
  a->row_tiles = ceil_div(d->a_rows, TM);
  a->a_pad = a->row_tiles * TM;
  a->col_tiles = (int)ceil_div64(a->n_cols > 0 ? a->n_cols : 1, TN);
  int splits = 2 * num_sms() / a->row_tiles;
  if (splits < 1) splits = 1;
  if (splits > a->col_tiles) splits = a->col_tiles;
  if (splits > num_sms()) splits = num_sms();
  a->splits = splits;
  return PCL_OK;
}

size_t pcl::simt_sweep_smem(int D, bool bwd, bool topk) {
  return (size_t)(2 * D * LDT + (bwd ? TM * LDT : 0)) * sizeof(float) + 64 * sizeof(void*) + 64 * 3 * sizeof(int) +
         64 * (topk ? 12 : 8) * sizeof(float);
}

extern "C" int pcl_sweep_sizes(const pcl_sweep_desc* d, pcl_sweep_sizes_t* out) {
  SweepArgs a;
  // pointers are not needed to size the buffers: validate the shape fields only
  pcl_sweep_desc tmp = *d;
  static const float dummy_f = 0.f;
  static const int32_t dummy_i = 0;
  tmp.anchors = &dummy_f; tmp.anchor_cls = &dummy_i;
  if (tmp.mode == 1) { tmp.segment_queue = &dummy_f; tmp.pixel_queue = &dummy_f; }
  if (tmp.mode == 2) { tmp.contrast = &dummy_f; tmp.contrast_cls = &dummy_i; }
  int st = simt_make_args(&tmp, &a);
  if (st != PCL_OK || !out) return st != PCL_OK ? st : PCL_ERR_ARG;
  out->n_real_cols = a.n_cols;
  out->row_tiles = a.row_tiles;
  out->splits = a.splits;
  out->partial_f32 = (int64_t)a.splits * a.a_pad;
  out->rowstat_f32 = a.a_rows;
  out->dpartial_f32 = (int64_t)a.splits * a.a_pad * a.D;
  return PCL_OK;
}

static TopkArgs topk_args(const SweepArgs& a, int k, uint32_t* scratch) {
  TopkArgs tk;
  tk.k = k;
  tk.hist = scratch;
  tk.sel = scratch + (int64_t)a.a_pad * TK_BINS;
  return tk;
}

extern "C" int pcl_infonce_fwd(const pcl_sweep_desc* d, float* partials, float* rowstats, float* loss, void* stream) {
  return pcl::simt_fwd_ex(d, 0, nullptr, partials, rowstats, loss, stream, nullptr);
}

extern "C" int pcl_infonce_bwd(const pcl_sweep_desc* d, const float* rowstats, const float* grad_loss,
                               float* dpartials, float* dA, void* stream) {
  return pcl::simt_bwd_ex(d, 0, nullptr, rowstats, grad_loss, dpartials, dA, stream);
}

// k == 0: all negatives (the reference).  k >= 1 (a10): the negative sum keeps the k hardest negatives of every anchor:
// three histogram sweeps with the warp-per-row scans of pcl_topk.cuh in between, then the weighted NEG sweep (the
// selection state stays in scratch for the backward); POS and finalize as usual.
int pcl::simt_fwd_ex(const pcl_sweep_desc* d, int k, uint32_t* scratch, float* partials, float* rowstats, float* loss,
                     void* stream, unsigned long long* step_counter) {
  SweepArgs a;
  int st = simt_make_args(d, &a);
  if (st != PCL_OK) return st;
  if (k < 0 || (k > 0 && !scratch)) return PCL_ERR_ARG;
  PCL_REQUIRE(partials && rowstats && loss);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = simt_sweep_smem(a.D, false, false);
  PCL_SMEM_OPT_IN(k_sweep<MODE_POS>, simt_sweep_smem(256, false, false));
  // every (split, live row) slot is written by its CTA (empty column ranges write "nothing seen"),
  // so the partial buffers need no initialisation
  dim3 grid(a.row_tiles, a.splits);
  if (k == 0) {
    PCL_SMEM_OPT_IN(k_sweep<MODE_NEG>, simt_sweep_smem(256, false, false));
    k_sweep<MODE_NEG><<<grid, SWEEP_THREADS, smem, s>>>(a, partials, nullptr, nullptr, TopkArgs{});
    PCL_LAUNCH_CHECK();
    k_combine_neg<false><<<ceil_div(a.a_rows, 256), 256, 0, s>>>(a, partials, rowstats, TopkArgs{});
    PCL_LAUNCH_CHECK();
  } else {
    const TopkArgs tk = topk_args(a, k, scratch);
    const size_t smem_tk = simt_sweep_smem(a.D, false, true);
    PCL_SMEM_OPT_IN(k_sweep<MODE_H1>, simt_sweep_smem(256, false, true));
    PCL_SMEM_OPT_IN(k_sweep<MODE_H2>, simt_sweep_smem(256, false, true));
    PCL_SMEM_OPT_IN(k_sweep<MODE_H3>, simt_sweep_smem(256, false, true));
    PCL_SMEM_OPT_IN(k_sweep<MODE_NEGW>, simt_sweep_smem(256, false, true));
    PCL_CUDA(cudaMemsetAsync(tk.hist, 0, (size_t)a.a_pad * TK_BINS * sizeof(uint32_t), s));
    const int scan_blocks = ceil_div(a.a_rows, 8);          // 8 warps (rows) per 256-thread block
    k_sweep<MODE_H1><<<grid, SWEEP_THREADS, smem_tk, s>>>(a, nullptr, nullptr, nullptr, tk);
    PCL_LAUNCH_CHECK();
    k_topk_scan<1><<<scan_blocks, 256, 0, s>>>(a, tk);
    PCL_LAUNCH_CHECK();
    k_sweep<MODE_H2><<<grid, SWEEP_THREADS, smem_tk, s>>>(a, nullptr, nullptr, nullptr, tk);
    PCL_LAUNCH_CHECK();
    k_topk_scan<2><<<scan_blocks, 256, 0, s>>>(a, tk);
    PCL_LAUNCH_CHECK();
    k_sweep<MODE_H3><<<grid, SWEEP_THREADS, smem_tk, s>>>(a, nullptr, nullptr, nullptr, tk);
    PCL_LAUNCH_CHECK();
    k_topk_scan<3><<<scan_blocks, 256, 0, s>>>(a, tk);
    PCL_LAUNCH_CHECK();
    k_sweep<MODE_NEGW><<<grid, SWEEP_THREADS, smem_tk, s>>>(a, partials, nullptr, nullptr, tk);
    PCL_LAUNCH_CHECK();
    k_combine_neg<true><<<ceil_div(a.a_rows, 256), 256, 0, s>>>(a, partials, rowstats, tk);
    PCL_LAUNCH_CHECK();
  }
  k_sweep<MODE_POS><<<grid, SWEEP_THREADS, smem, s>>>(a, partials, rowstats, nullptr, TopkArgs{});   // positives: no selection
  PCL_LAUNCH_CHECK();
  k_finalize<<<1, 1024, 0, s>>>(a, partials, rowstats, loss, step_counter);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

// k as in simt_fwd_ex; k >= 1 reads the selection state the forward left in scratch
int pcl::simt_bwd_ex(const pcl_sweep_desc* d, int k, uint32_t* scratch, const float* rowstats, const float* grad_loss,
                     float* dpartials, float* dA, void* stream) {
  SweepArgs a;
  int st = simt_make_args(d, &a);
  if (st != PCL_OK) return st;
  if (k < 0 || (k > 0 && !scratch)) return PCL_ERR_ARG;
  PCL_REQUIRE(rowstats && dpartials && dA);
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid(a.row_tiles, a.splits);
  if (k == 0) {
    PCL_SMEM_OPT_IN(k_sweep<MODE_BWD>, simt_sweep_smem(256, true, false));
    k_sweep<MODE_BWD><<<grid, SWEEP_THREADS, simt_sweep_smem(a.D, true, false), s>>>(a, nullptr, rowstats, dpartials,
                                                                                      TopkArgs{});
  } else {
    PCL_SMEM_OPT_IN(k_sweep<MODE_BWDW>, simt_sweep_smem(256, true, true));
    k_sweep<MODE_BWDW><<<grid, SWEEP_THREADS, simt_sweep_smem(a.D, true, true), s>>>(a, nullptr, rowstats, dpartials,
                                                                                      topk_args(a, k, scratch));
  }
  PCL_LAUNCH_CHECK();
  const int64_t total = (int64_t)a.a_rows * a.D;
  k_reduce_dA<<<(unsigned)ceil_div64(total, 256), 256, 0, s>>>(a, dpartials, grad_loss, dA);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}
