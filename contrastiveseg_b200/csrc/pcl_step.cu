// One loss step chained on a stream behind a single descriptor (include/pcl.h: pcl_step_*).
#include "pcl_common.cuh"
#include <stdlib.h>

static void fill_sweep(const pcl_step_desc* d, pcl_sweep_desc* w) {
  memset(w, 0, sizeof(*w));
  const int ms = d->g.max_samples;
  w->anchors = d->anchors_f32;
  w->anchor_cls = d->anchor_meta + 2 * (int64_t)ms;
  w->diag_col = d->anchor_meta + 3 * (int64_t)ms;       // reference row index r = v*TC + t (Q1)
  w->plan = d->plan;
  w->a_rows = ms;
  w->D = d->g.D;
  w->mode = d->mode;
  w->segment_queue = d->segment_queue;
  w->pixel_queue = d->pixel_queue;
  w->bank_K = d->bank_K; w->bank_M0 = d->bank_M0; w->bank_M1 = d->bank_M1;
  w->temperature = d->temperature; w->base_temperature = d->base_temperature;
  w->nan_safe = d->nan_safe;
}

static void fill_tc(const pcl_step_desc* d, pcl_tc_desc* t) {
  memset(t, 0, sizeof(*t));
  const int ms = d->g.max_samples;
  t->anchors_f32 = nullptr;                              // bf16 rows were written by pcl_select_gather
  t->anchors_bf16 = d->anchors_bf16;
  t->anchor_cls = d->anchor_meta + 2 * (int64_t)ms;
  t->diag_col = d->anchor_meta + 3 * (int64_t)ms;
  t->plan = d->plan;
  t->a_rows = ms;
  t->D = d->g.D;
  t->mode = d->mode;
  t->contrast_bf16 = d->shadow_bf16;
  t->contrast_rows_alloc = d->shadow_rows;
  t->bank_K = d->bank_K;
  t->bank_R = d->bank_M0 + d->bank_M1;
  t->sorted = 1;
  t->contrast_norm_bound = d->contrast_norm_bound;
  t->temperature = d->temperature; t->base_temperature = d->base_temperature;
  t->nan_safe = d->nan_safe;
}

extern "C" int pcl_step_stats(const pcl_step_desc* d, void* stream) {
  if (!d) return PCL_ERR_ARG;
  if (d->sync != nullptr)        // one launch: the scan's last block computes totals and plan (sync[4] = its counter)
    return pcl::class_stats_plan(&d->g, d->labels, d->seg, d->predict, d->keys, d->chunk_pref, d->counts, d->plan,
                                 d->sync + 4, stream);
  int st = pcl_class_stats(&d->g, d->labels, d->seg, d->predict, d->keys, d->chunk_pref, d->counts, stream);
  if (st != PCL_OK) return st;
  return pcl_plan_anchors(&d->g, d->counts, d->plan, stream);
}

static int step_forward(const pcl_step_desc* d, unsigned long long* ctr, void* stream);

extern "C" int pcl_step_forward(const pcl_step_desc* d, void* stream) { return step_forward(d, nullptr, stream); }

// Captured sequences: the anchors are drawn by the selection kernel itself from *step_counter (same keyed bijection and
// seed formula as pcl_step_ranks, whose single CTA needed 13-15 us for 1024 draws) and the forward's last kernel advances
// the counter — no separate rank-draw launch.
extern "C" int pcl_step_forward_ctr(const pcl_step_desc* d, uint64_t* step_counter, void* stream) {
  if (!step_counter) return PCL_ERR_ARG;
  return step_forward(d, reinterpret_cast<unsigned long long*>(step_counter), stream);
}

static int step_forward(const pcl_step_desc* d, unsigned long long* ctr, void* stream) {
  if (!d) return PCL_ERR_ARG;
  if (d->precision == 1) {
    // tensor path: the selection kernel also writes the row stabilisers and initialises the partial slots
    if (!d->anchors_bf16 || !d->row_m2 || (d->mode == 1 && !d->shadow_bf16)) return PCL_ERR_ARG;
    pcl_tc_desc t;
    fill_tc(d, &t);
    int64_t n_slot_rows = 0;
    float m2_scale = 0.f;
    int st = pcl::tc_query(&t, &n_slot_rows, &m2_scale);
    if (st != PCL_OK) return st;
    st = pcl::select_gather_ex(&d->g, d->embed, d->keys, d->chunk_pref, d->plan, ctr ? nullptr : d->ranks, d->seed,
                               d->normalize, d->anchor_meta, d->anchors_f32, d->anchors_bf16, d->inv_norm, nullptr, d->row_m2,
                               m2_scale, d->partials, n_slot_rows, stream, ctr);
    if (st != PCL_OK) return st;
    return pcl::tc_fwd_ex(&t, d->row_m2, d->partials, d->rowstats, d->loss, stream, true, ctr);
  }
  int st = pcl::select_gather_ex(&d->g, d->embed, d->keys, d->chunk_pref, d->plan, ctr ? nullptr : d->ranks, d->seed,
                                 d->normalize, d->anchor_meta, d->anchors_f32, d->anchors_bf16, d->inv_norm, d->norm_max,
                                 nullptr, 0.f, nullptr, 0, stream, ctr);
  if (st != PCL_OK) return st;
  pcl_sweep_desc w;
  fill_sweep(d, &w);
  return pcl::simt_fwd_ex(&w, d->partials, d->rowstats, d->loss, stream, ctr);
}

extern "C" int pcl_step_backward(const pcl_step_desc* d, const float* grad_loss, void* stream) {
  if (!d) return PCL_ERR_ARG;
  int st;
  if (d->precision == 1) {
    pcl_tc_desc t;
    fill_tc(d, &t);
    if (!d->normalize) {
      // fused tail: the dense-gradient writer sums the per-split partials itself (no (A, D) gradient round trip)
      int splits = 0, a_pad = 0;
      st = pcl::tc_bwd_ex(&t, d->row_m2, d->rowstats, grad_loss, d->dpartials, nullptr, stream, &splits, &a_pad);
      if (st != PCL_OK) return st;
      return pcl::zero_scatter_reduce(&d->g, d->plan, d->anchor_meta, d->dpartials, splits, a_pad, 1.f / d->temperature,
                                      grad_loss, d->grad_embed, stream);
    }
    st = pcl_infonce_tc_bwd(&t, d->row_m2, d->rowstats, grad_loss, d->dpartials, d->dA, stream);
  } else {
    pcl_sweep_desc w;
    fill_sweep(d, &w);
    st = pcl_infonce_bwd(&w, d->rowstats, grad_loss, d->dpartials, d->dA, stream);
  }
  if (st != PCL_OK) return st;
  return pcl_scatter_grad(&d->g, d->plan, d->anchor_meta, d->dA, d->anchors_f32, d->inv_norm, d->normalize,
                          d->grad_embed, stream);
}

// Backward for a dense-gradient buffer the caller has ALREADY zero-filled (the 268 MB fill is the HBM floor of the
// step; a caller that starts it on a second stream at the beginning of the forward hides it behind the latency-bound
// selection and sweep kernels): backward sweep -> (A, D) gradient rows -> scatter of those rows only.
extern "C" int pcl_step_backward_prezeroed(const pcl_step_desc* d, const float* grad_loss, void* stream) {
  if (!d) return PCL_ERR_ARG;
  int st;
  if (d->precision == 1) {
    pcl_tc_desc t;
    fill_tc(d, &t);
    if (!d->normalize) {
      // the scatter sums the per-split partial rows itself (fixed order): no (A, D) gradient round trip, one launch less
      int splits = 0, a_pad = 0;
      st = pcl::tc_bwd_ex(&t, d->row_m2, d->rowstats, grad_loss, d->dpartials, nullptr, stream, &splits, &a_pad);
      if (st != PCL_OK) return st;
      return pcl::scatter_reduce_rows(&d->g, d->plan, d->anchor_meta, d->dpartials, splits, 0, a_pad, 1.f / d->temperature,
                                      grad_loss, d->grad_embed, nullptr, stream, d->sync);
    }
    st = pcl_infonce_tc_bwd(&t, d->row_m2, d->rowstats, grad_loss, d->dpartials, d->dA, stream);
  } else {
    pcl_sweep_desc w;
    fill_sweep(d, &w);
    st = pcl_infonce_bwd(&w, d->rowstats, grad_loss, d->dpartials, d->dA, stream);
  }
  if (st != PCL_OK) return st;
  return pcl::scatter_rows(&d->g, d->plan, d->anchor_meta, d->dA, d->anchors_f32, d->inv_norm, d->normalize,
                           d->grad_embed, stream);
}

// ---- fused small-anchor step (include/pcl.h: pcl_step_fused_*) ----
extern "C" int pcl_step_fused_supported(const pcl_step_desc* d) {
  if (!d || d->mode != 0 || d->precision != 1 || d->normalize != 0 || d->sync == nullptr) return 0;
  if (d->g.D != 256 || d->g.max_samples < 1 || d->g.max_samples > 1024) return 0;
  return 1;
}

extern "C" int pcl_step_fused_select(const pcl_step_desc* d, const uint64_t* step_counter, const int32_t* prev_rows,
                                     void* stream) {
  if (!pcl_step_fused_supported(d)) return PCL_ERR_UNSUPPORTED;
  if (!d->anchors_bf16 || !d->row_m2 || (prev_rows && !d->grad_embed)) return PCL_ERR_ARG;
  pcl_tc_desc t;
  fill_tc(d, &t);
  int64_t n_slot_rows = 0;
  float m2_scale = 0.f;
  int st = pcl::tc_query(&t, &n_slot_rows, &m2_scale);
  if (st != PCL_OK) return st;
  // selection + gather; the fused kernel writes every partial slot it reads: no slot initialisation
  return pcl::select_gather_ex(&d->g, d->embed, d->keys, d->chunk_pref, d->plan, step_counter ? nullptr : d->ranks, d->seed,
                               0, d->anchor_meta, d->anchors_f32, d->anchors_bf16, d->inv_norm, nullptr, d->row_m2, m2_scale,
                               nullptr, 0, stream, reinterpret_cast<const unsigned long long*>(step_counter), d->sync,
                               prev_rows, d->grad_embed);
}

extern "C" int pcl_step_fused_loss(const pcl_step_desc* d, void* stream) {
  if (!pcl_step_fused_supported(d)) return PCL_ERR_UNSUPPORTED;
  if (!d->anchors_bf16 || !d->row_m2) return PCL_ERR_ARG;
  pcl_tc_desc t;
  fill_tc(d, &t);
  return pcl::self_fused(&t, d->row_m2, d->partials, d->rowstats, d->loss, d->dpartials, d->sync, stream);
}

extern "C" int pcl_step_fused_scatter(const pcl_step_desc* d, const float* grad_scale, uint64_t* step_counter,
                                      int32_t* prev_rows, void* stream) {
  if (!pcl_step_fused_supported(d)) return PCL_ERR_UNSUPPORTED;
  if (!d->grad_embed) return PCL_ERR_ARG;
  const int a_pad = ((d->g.max_samples + 127) / 128) * 128;
  const int splits = (a_pad + 255) / 256;
  return pcl::scatter_reduce_rows(&d->g, d->plan, d->anchor_meta, d->dpartials, splits, 256, a_pad, 1.f / d->temperature, grad_scale,
                                  d->grad_embed, reinterpret_cast<unsigned long long*>(step_counter), stream, d->sync, prev_rows);
}

// zero-fill of the step's dense gradient on the engine's fill kernel (the caller picks the stream: a parallel branch)
extern "C" int pcl_step_fused_fill(const pcl_step_desc* d, void* stream) {
  if (!d || !d->grad_embed) return PCL_ERR_ARG;
  const uint64_t bytes = (uint64_t)d->g.B * d->g.D * d->g.h * d->g.w * sizeof(float);
  if ((bytes & 15) != 0 || ((uintptr_t)d->grad_embed & 15) != 0) return PCL_ERR_UNSUPPORTED;
  // The fill forks right before the fused InfoNCE kernel (at most 8 x 4 = 32 CTAs, one per SM).  Its CTAs OWN their SMs
  // and leave 32 free: the InfoNCE kernel starts at once, next to the fill, instead of waiting for fill CTAs to retire
  // (its 384-thread, register-heavy CTAs fit on no SM that holds fill warps).  PCL_FILL_RESERVE_SMS overrides (tuning
  // runs; 0 = the shared-SM fill).
  int reserve = 32;
  if (const char* e = getenv("PCL_FILL_RESERVE_SMS")) reserve = atoi(e);
  return pcl::fill_zero(d->grad_embed, bytes, stream, d->sync, reserve);
}
