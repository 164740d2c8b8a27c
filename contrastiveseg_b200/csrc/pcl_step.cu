// One loss step chained on a stream behind a single descriptor (include/pcl.h: pcl_step_*).
#include "pcl_common.cuh"

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
  // with the sync buffer: one launch, the scan's last block computes totals and plan (sync[4] = its counter)
  unsigned int* done_ctr = d->sync != nullptr ? d->sync + 4 : nullptr;
  int st = pcl::class_stats(&d->g, d->labels, d->seg, d->predict, d->keys, d->chunk_pref, d->counts, d->plan, done_ctr,
                            stream, d->seg_dtype);
  if (st != PCL_OK || done_ctr != nullptr) return st;
  return pcl_plan_anchors(&d->g, d->counts, d->plan, stream);
}

// a10: topk_negatives 0 = all negatives, k >= 1 needs the selection scratch, < 0 is refused
static bool topk_ok(const pcl_step_desc* d) {
  return d->topk_negatives == 0 || (d->topk_negatives > 0 && d->topk_scratch != nullptr);
}

// The selection's arguments that come from the descriptor; ctr: captured sequences draw the anchors from the counter
// instead of the injected ranks.  The caller sets the rest.
static pcl::select_args select_args(const pcl_step_desc* d, const unsigned long long* ctr) {
  pcl::select_args a = {};
  a.g = &d->g; a.embed = d->embed; a.embed_dtype = d->embed_dtype;
  a.keys = d->keys; a.chunk_pref = d->chunk_pref; a.plan = d->plan; a.ranks = ctr ? nullptr : d->ranks;
  a.seed = d->seed; a.normalize = d->normalize; a.seed_ctr = ctr;
  a.anchor_meta = d->anchor_meta; a.anchors_f32 = d->anchors_f32; a.anchors_bf16 = d->anchors_bf16; a.inv_norm = d->inv_norm;
  return a;
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
  if (!d || !topk_ok(d)) return PCL_ERR_ARG;
  const int k = d->topk_negatives;
  pcl::select_args sel = select_args(d, ctr);
  if (d->precision == 1 && k == 0) {
    // tensor path: the selection kernel also writes the row stabilisers and initialises the partial slots
    if (!d->anchors_bf16 || !d->row_m2 || (d->mode == 1 && !d->shadow_bf16)) return PCL_ERR_ARG;
    pcl_tc_desc t;
    fill_tc(d, &t);
    int st = pcl::tc_query(&t, &sel.n_slot_rows, &sel.m2_scale);
    if (st != PCL_OK) return st;
    sel.row_m2 = d->row_m2;
    sel.partials = d->partials;
    st = pcl::select_gather(sel, stream);
    if (st != PCL_OK) return st;
    return pcl::tc_fwd_ex(&t, d->row_m2, d->partials, d->rowstats, d->loss, stream, true, ctr);
  }
  sel.norm_max = d->norm_max;
  int st = pcl::select_gather(sel, stream);
  if (st != PCL_OK) return st;
  if (d->precision == 1) {
    // top-k on the tensor path: the selection above leaves the stabilisers and the partial slots to the top-k forward's
    // own prep (k_select would round the stabiliser differently: sqrt * (cbound * k1 * 1.0001) against
    // ((sqrt * cbound) * k1) * 1.0001 in k_tc_prep)
    pcl_tc_desc t;
    fill_tc(d, &t);
    return pcl::tc_fwd_topk_ex(&t, k, d->topk_scratch, d->row_m2, d->partials, d->rowstats, d->loss, stream, false, ctr);
  }
  pcl_sweep_desc w;
  fill_sweep(d, &w);
  return pcl::simt_fwd_ex(&w, k, d->topk_scratch, d->partials, d->rowstats, d->loss, stream, ctr);
}

// The backward sweep of the step (the top-k one with topk_negatives); *r = where the anchor rows of the gradient are.
static int step_sweep_bwd(const pcl_step_desc* d, const float* grad_loss, void* stream, pcl::grad_rows* r) {
  if (!topk_ok(d)) return PCL_ERR_ARG;
  const int k = d->topk_negatives;
  // tensor path without normalise and top-k: the sweep leaves its per-split partial rows and the gradient writer sums
  // them itself (fixed order), no (A, D) gradient round trip; otherwise the sweep reduces them to dA
  const bool partial_rows = d->precision == 1 && !d->normalize && k == 0;
  *r = {};
  if (partial_rows) {
    r->dpartials = d->dpartials; r->inv_T = 1.f / d->temperature; r->grad_scale = grad_loss;
  } else {
    r->dA = d->dA; r->anchors_f32 = d->anchors_f32; r->inv_norm = d->inv_norm; r->normalize = d->normalize;
  }
  if (d->precision == 1) {
    pcl_tc_desc t;
    fill_tc(d, &t);
    return pcl::tc_bwd_ex(&t, d->row_m2, d->rowstats, grad_loss, d->dpartials, partial_rows ? nullptr : d->dA, stream,
                          &r->splits, &r->a_pad, k > 0 ? d->topk_scratch : nullptr);
  }
  pcl_sweep_desc w;
  fill_sweep(d, &w);
  return pcl::simt_bwd_ex(&w, k, d->topk_scratch, d->rowstats, grad_loss, d->dpartials, d->dA, stream);
}

// prezeroed: the caller has ALREADY zero-filled the dense gradient (the 268 MB fill is the HBM floor of the step; a
// caller that starts it on a second stream at the beginning of the forward hides it behind the latency-bound selection
// and sweep kernels), so only the anchor rows are scattered.
static int step_backward(const pcl_step_desc* d, const float* grad_loss, void* stream, bool prezeroed) {
  if (!d) return PCL_ERR_ARG;
  if (prezeroed && d->topk_negatives != 0) return PCL_ERR_UNSUPPORTED;
  pcl::grad_rows r;
  int st = step_sweep_bwd(d, grad_loss, stream, &r);
  if (st != PCL_OK) return st;
  return pcl::dense_grad(&d->g, d->plan, d->anchor_meta, r, prezeroed, d->grad_embed, d->embed_dtype, stream, d->sync);
}

extern "C" int pcl_step_backward(const pcl_step_desc* d, const float* grad_loss, void* stream) {
  return step_backward(d, grad_loss, stream, false);
}

extern "C" int pcl_step_backward_prezeroed(const pcl_step_desc* d, const float* grad_loss, void* stream) {
  return step_backward(d, grad_loss, stream, true);
}

// The backward with the anchor columns as its output instead of the dense gradient (grad_embed is not touched)
extern "C" int pcl_step_backward_cols(const pcl_step_desc* d, const float* grad_loss, float* cols, int32_t* col_pix,
                                      void* stream) {
  if (!d || !cols || !col_pix) return PCL_ERR_ARG;
  pcl::grad_rows r;
  int st = step_sweep_bwd(d, grad_loss, stream, &r);
  if (st != PCL_OK) return st;
  return pcl::anchor_cols(&d->g, d->plan, d->anchor_meta, r, cols, col_pix, stream);
}

// ---- fused small-anchor step (include/pcl.h: pcl_step_fused_*) ----
extern "C" int pcl_step_fused_supported(const pcl_step_desc* d) {
  if (!d || d->mode != 0 || d->precision != 1 || d->normalize != 0 || d->sync == nullptr || d->topk_negatives != 0) return 0;
  if (d->g.D != 256 || d->g.max_samples < 1 || d->g.max_samples > 1024) return 0;
  if (!pcl::dtype_ok(d->embed_dtype) || !pcl::dtype_ok(d->seg_dtype)) return 0;      // fp32, bf16 and fp16 inputs qualify
  return 1;
}

extern "C" int pcl_step_fused_select(const pcl_step_desc* d, const uint64_t* step_counter, const int32_t* prev_rows,
                                     void* stream) {
  if (!pcl_step_fused_supported(d)) return PCL_ERR_UNSUPPORTED;
  if (!d->anchors_bf16 || !d->row_m2 || (prev_rows && !d->grad_embed)) return PCL_ERR_ARG;
  pcl_tc_desc t;
  fill_tc(d, &t);
  // selection + gather; the fused kernel writes every partial slot it reads: no slot initialisation
  pcl::select_args sel = select_args(d, reinterpret_cast<const unsigned long long*>(step_counter));
  int st = pcl::tc_query(&t, &sel.n_slot_rows, &sel.m2_scale);     // (no partials: the slot count goes unused)
  if (st != PCL_OK) return st;
  sel.row_m2 = d->row_m2;
  sel.dbg = d->sync;
  sel.prev_rows = prev_rows;
  sel.grad_clear = d->grad_embed;
  return pcl::select_gather(sel, stream);
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
  pcl::grad_rows r = {};
  pcl::self_fused_splits(d->g.max_samples, &r.a_pad, &r.splits, &r.split_cols);
  r.dpartials = d->dpartials;
  r.inv_T = 1.f / d->temperature;
  r.grad_scale = grad_scale;
  return pcl::dense_grad(&d->g, d->plan, d->anchor_meta, r, true, d->grad_embed, d->embed_dtype, stream, d->sync,
                         reinterpret_cast<unsigned long long*>(step_counter), prev_rows);
}

// The fused step's anchor columns in place of the scatter: the same partial sums, no dense gradient
extern "C" int pcl_step_fused_cols(const pcl_step_desc* d, const float* grad_scale, uint64_t* step_counter, float* cols,
                                   int32_t* col_pix, void* stream) {
  if (!pcl_step_fused_supported(d)) return PCL_ERR_UNSUPPORTED;
  if (!cols || !col_pix) return PCL_ERR_ARG;
  pcl::grad_rows r = {};
  pcl::self_fused_splits(d->g.max_samples, &r.a_pad, &r.splits, &r.split_cols);
  r.dpartials = d->dpartials;
  r.inv_T = 1.f / d->temperature;
  r.grad_scale = grad_scale;
  return pcl::anchor_cols(&d->g, d->plan, d->anchor_meta, r, cols, col_pix, stream,
                          reinterpret_cast<unsigned long long*>(step_counter));
}

// zero-fill of the step's dense gradient on the engine's fill kernel (the caller picks the stream: a parallel branch)
extern "C" int pcl_step_fused_fill(const pcl_step_desc* d, void* stream) {
  if (!d || !d->grad_embed || !pcl::dtype_ok(d->embed_dtype)) return PCL_ERR_ARG;
  if (d->topk_negatives != 0) return PCL_ERR_UNSUPPORTED;
  // sized by the gradient's element size: a half gradient is half the bytes (still a multiple of 16: D % 32 == 0)
  const uint64_t bytes = (uint64_t)d->g.B * d->g.D * d->g.h * d->g.w * pcl::dtype_size(d->embed_dtype);
  if ((bytes & 15) != 0 || ((uintptr_t)d->grad_embed & 15) != 0) return PCL_ERR_UNSUPPORTED;
  // The fill forks right before the fused InfoNCE kernel (at most 8 x 4 = 32 CTAs, one per SM).  Its CTAs OWN their SMs
  // and leave 32 free: the InfoNCE kernel starts at once, next to the fill, instead of waiting for fill CTAs to retire
  // (its 384-thread, register-heavy CTAs fit on no SM that holds fill warps; measured in-graph on H100 with the
  // shared-SM fill: the fused kernel starts 58 us later, step 0.164 -> 0.191 ms).
  return pcl::fill_zero(d->grad_embed, bytes, stream, d->sync, 32);
}
