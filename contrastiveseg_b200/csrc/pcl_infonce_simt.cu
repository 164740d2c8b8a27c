// Exact-fp32 InfoNCE sweep (SURVEY §8 rows a5, a6) — SIMT tiles, no A x N temporaries.
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
#include "pcl_common.cuh"
#include "pcl_sweep.cuh"
#include "pcl_simt_tile.cuh"

namespace pcl {

enum { MODE_NEG = 0, MODE_POS = 1, MODE_BWD = 2 };

template <int MODE>
__global__ void __launch_bounds__(SWEEP_THREADS, 1)
k_sweep(SweepArgs a, float* __restrict__ partials, const float* __restrict__ rowstats, float* __restrict__ dpartials) {
  extern __shared__ __align__(16) float smem[];
  const int D = a.D;
  float* As_t = smem;                         // [D][LDT]
  float* Ct = As_t + D * LDT;                 // [D][LDT]
  float* Gs = Ct + D * LDT;                   // [TM][LDT]   (BWD only)
  float* s_extra = Gs + (MODE == MODE_BWD ? TM * LDT : 0);
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
    if (MODE != MODE_NEG) {
      const float* st = rowstats;
      s_rm[tid] = ok ? st[r] : 0.f;
      s_rneg[tid] = ok ? st[a.a_rows + r] : 1.f;
      if (MODE == MODE_BWD) {
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
  for (int i = 0; i < 4; ++i) { run_m[i] = MODE == MODE_NEG ? -CUDART_INF_F : 0.f; run_a[i] = 0.f; run_b[i] = 0.f; }
  float dacc[4][QMAX];
  if (MODE == MODE_BWD) {
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
      if (MODE == MODE_BWD && a.mode == 0) {
        bool ok = n < ncols;
        s_cm[tid] = ok ? rowstats[n] : 0.f;
        s_cneg[tid] = ok ? rowstats[a.a_rows + n] : 1.f;
        s_cs[tid] = ok ? rowstats[3 * a.a_rows + n] : 0.f;
        float np = ok ? rowstats[4 * a.a_rows + n] : 1.f;
        float c = rs_scale / np;
        if (a.nan_safe && !(np > 0.f)) c = 0.f;
        s_cc[tid] = ok ? c : 0.f;
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
    if (MODE == MODE_NEG) {
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
      // gradient tile G (closed form, SURVEY appendix A)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = ty * 4 + i;
        const int rcls = s_rcls[r], rdiag = s_rdiag[r];
        const float m = s_rm[r], neg = s_rneg[r], S = s_rs[r], c = s_rc[r];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cj = tx * 4 + j;
          const int lab = s_clab[cj];
          float gval = 0.f;
          if (lab != -2 && rcls >= 0) {
            const float l = acc[i][j] * a.inv_T;
            const float e = expf(l - m);
            if (lab == rcls) {
              if ((col_base + j) != (int64_t)rdiag) gval = -c * (1.f - e / (e + neg));
            } else {
              gval = c * e * S;
            }
            if (a.mode == 0) {               // + G_ji: the column is an anchor too (self-contrast)
              const float e2 = expf(l - s_cm[cj]);
              if (lab == rcls) {
                if ((col_base + j) != (int64_t)rdiag) gval += -s_cc[cj] * (1.f - e2 / (e2 + s_cneg[cj]));
              } else {
                gval += s_cc[cj] * e2 * s_cs[cj];
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

  // ---- write partials ----
  if (MODE == MODE_NEG) {
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
  } else {
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

size_t pcl::simt_sweep_smem(int D, bool bwd) {
  return (size_t)(2 * D * LDT + (bwd ? TM * LDT : 0)) * sizeof(float) + 64 * sizeof(void*) + 64 * 3 * sizeof(int) +
         64 * 8 * sizeof(float);
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

extern "C" int pcl_infonce_fwd(const pcl_sweep_desc* d, float* partials, float* rowstats, float* loss, void* stream) {
  return pcl::simt_fwd_ex(d, partials, rowstats, loss, stream, nullptr);
}

int pcl::simt_fwd_ex(const pcl_sweep_desc* d, float* partials, float* rowstats, float* loss, void* stream,
                     unsigned long long* step_counter) {
  SweepArgs a;
  int st = simt_make_args(d, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(partials && rowstats && loss);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = simt_sweep_smem(a.D, false);
  PCL_SMEM_OPT_IN(k_sweep<MODE_NEG>, simt_sweep_smem(256, false));
  PCL_SMEM_OPT_IN(k_sweep<MODE_POS>, simt_sweep_smem(256, false));
  // every (split, live row) slot is written by its CTA (empty column ranges write "nothing seen"),
  // so the partial buffers need no initialisation
  dim3 grid(a.row_tiles, a.splits);
  k_sweep<MODE_NEG><<<grid, SWEEP_THREADS, smem, s>>>(a, partials, nullptr, nullptr);
  PCL_LAUNCH_CHECK();
  k_combine_neg<<<ceil_div(a.a_rows, 256), 256, 0, s>>>(a, partials, rowstats);
  PCL_LAUNCH_CHECK();
  k_sweep<MODE_POS><<<grid, SWEEP_THREADS, smem, s>>>(a, partials, rowstats, nullptr);
  PCL_LAUNCH_CHECK();
  k_finalize<<<1, 1024, 0, s>>>(a, partials, rowstats, loss, step_counter);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

int pcl::simt_launch_pos(const SweepArgs& a, float* partials, const float* rowstats, cudaStream_t s) {
  const size_t smem = simt_sweep_smem(a.D, false);
  // (round 1 set the limit to THIS call's size here: a D=64 top-k call lowered it under the D=256 size the forward
  // believed to be in place -> cudaErrorInvalidValue on the next D=256 POS launch.  Now: one opt-in to the maximum.)
  PCL_SMEM_OPT_IN(k_sweep<MODE_POS>, simt_sweep_smem(256, false));
  dim3 grid(a.row_tiles, a.splits);
  k_sweep<MODE_POS><<<grid, SWEEP_THREADS, smem, s>>>(a, partials, rowstats, nullptr);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_infonce_bwd(const pcl_sweep_desc* d, const float* rowstats, const float* grad_loss,
                               float* dpartials, float* dA, void* stream) {
  SweepArgs a;
  int st = simt_make_args(d, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(rowstats && dpartials && dA);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = simt_sweep_smem(a.D, true);
  PCL_SMEM_OPT_IN(k_sweep<MODE_BWD>, simt_sweep_smem(256, true));
  dim3 grid(a.row_tiles, a.splits);
  k_sweep<MODE_BWD><<<grid, SWEEP_THREADS, smem, s>>>(a, nullptr, rowstats, dpartials);
  PCL_LAUNCH_CHECK();
  const int64_t total = (int64_t)a.a_rows * a.D;
  k_reduce_dA<<<(unsigned)ceil_div64(total, 256), 256, 0, s>>>(a, dpartials, grad_loss, dA);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}
