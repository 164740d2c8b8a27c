/*
 * pcl.h — C ABI of the H100 pixel-contrast loss engine (libpcl_b200.so).
 *
 * The reference (tfzhou/ContrastiveSeg) has no FFI on this path: it is Python/ATen behind three
 * nn.Module classes and one trainer method (SURVEY.md §8b).  This header is the boundary a
 * maintainer binds instead; each entry point names the reference code it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller unless the name starts with h_;
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), re-entrant and never throws; the
 *     library keeps no state between calls (apart from a mutex-protected cache of encoded TMA descriptors, which
 *     describe addresses/shapes only); the return value is 0 or a negative pcl_status;
 *   - scratch comes from caller-provided buffers (sizes: pcl_select_sizes / pcl_sweep_sizes), so the
 *     caller's allocator owns all memory and the sequence is CUDA-graph capturable;
 *   - there is NO CPU fallback: without a CUDA device every compute call returns PCL_ERR_CUDA;
 *   - one device per process (the one-process-per-GPU model of the reference's DDP launcher,
 *     lib/utils/distributed.py): opt-in shared-memory limits are raised once per process with cudaFuncSetAttribute,
 *     which is a per-device setting, so driving a second device from the same process is not supported.
 */
#ifndef PCL_H_
#define PCL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCL_VERSION 100          /* major*100 + minor */
#define PCL_MAX_CLASSES 256      /* class ids tracked: [0, K), K <= 256 */
#define PCL_CHUNK 1024           /* pixels per selection chunk */
#define PCL_ROW_TILE 64          /* anchor rows per SIMT tile */
#define PCL_PLAN_HEADER 16       /* int32 words at the start of the plan buffer */

typedef enum {
  PCL_OK = 0,
  PCL_ERR_ARG = -1,        /* bad argument (null pointer, size out of range, unsupported D ...) */
  PCL_ERR_CUDA = -2,       /* CUDA runtime error (see pcl_last_cuda_error) or no device */
  PCL_ERR_UNSUPPORTED = -3,/* valid request the engine does not implement (e.g. tensor path with D != 256) */
  PCL_ERR_SHAPE = -4       /* reference would raise an index error (e.g. Q6 label grid larger than feature map) */
} pcl_status;

/* plan buffer header words (int32), written by pcl_plan_anchors */
enum { PCL_PLAN_TC = 0, PCL_PLAN_V = 1, PCL_PLAN_A = 2, PCL_PLAN_FLAGS = 3, PCL_PLAN_NPAIR_MAX = 4 };
/* PCL_PLAN_FLAGS bits */
enum { PCL_FLAG_NO_CLASS = 1, PCL_FLAG_ZERO_VIEWS = 2, PCL_FLAG_SPLIT_ERROR = 4 };
/* Element type of an input that may be half precision (pcl_step_desc.embed_dtype / seg_dtype, pcl_bank_packet_dt).
 * Half inputs are converted to fp32 on load (exact) and everything downstream computes in fp32 as for fp32 inputs; a
 * half dense gradient is the fp32 gradient rounded once to nearest-even. */
enum { PCL_DT_F32 = 0, PCL_DT_BF16 = 1, PCL_DT_F16 = 2 };

int         pcl_version(void);
const char* pcl_strerror(int status);
const char* pcl_last_cuda_error(void);          /* text of the last CUDA error seen by this thread */
int         pcl_device_count(void);             /* 0 without a usable CUDA device */
/* FFI layout self-check: sizeof() of a host struct as this library was compiled.  struct_id: 0 pcl_geom,
 * 1 pcl_select_sizes_t, 2 pcl_sweep_desc, 3 pcl_sweep_sizes_t, 4 pcl_bank_geom, 5 pcl_tc_desc, 6 pcl_step_desc;
 * -1 for an unknown id.  A binding compares these with its own struct definitions before the first call. */
int64_t     pcl_abi_sizeof(int struct_id);
/* Diagnostics: number of kernels this library has launched (or recorded into a stream capture) since it was loaded,
 * process-wide.  The difference around one eager pass of a call sequence = kernels per step (bench.py: gpu_launches). */
uint64_t    pcl_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Geometry of one loss call (host struct, passed by pointer).
 * ----------------------------------------------------------------------------------------------*/
typedef struct {
  int32_t B, D, h, w;          /* embedding (B,D,h,w) fp32 NCHW; D % 32 == 0 and D <= 256        */
  int32_t Himg, Wimg;          /* label map (B,Himg,Wimg) int64                                  */
  int32_t K;                   /* number of class ids, labels outside [0,K) count as ignored     */
  int32_t max_samples;         /* contrast.max_samples                                            */
  int32_t max_views;           /* contrast.max_views                                              */
  int32_t ignore_label;        /* loss.params.ce_ignore_index (default -1)                        */
} pcl_geom;

/* Element counts of the selection scratch buffers for a geometry. */
typedef struct {
  int64_t keys_u16;            /* B*h*w             uint16 pixel keys (2*label + easy, 2K = ignored) */
  int64_t chunk_pref_i32;      /* B*2K*nchunk       per-chunk histogram of the pixel keys           */
  int64_t counts_i32;          /* B*2K              per-image key totals                            */
  int64_t plan_i32;            /* header + 8 words per (image,class) pair                           */
  int64_t anchor_meta_i32;     /* 4*max_samples     pixel, image, class, reference row              */
  int32_t nchunk;
  int32_t max_pairs;           /* B*K */
} pcl_select_sizes_t;

int pcl_select_sizes(const pcl_geom* g, pcl_select_sizes_t* out);

/* ------------------------------------------------------------------------------------------------
 * a3 + a4 (first half): label down-sampling, argmax, hard/easy key per pixel, per-chunk histograms.
 * Replaces lib/loss/loss_contrast.py:131-134 (nearest interpolation of the label map),
 * :183 (torch.max(seg,1)) and the unique/nonzero scans of :37-39,:60-61.
 *   labels   (B,Himg,Wimg) int64
 *   seg      (B,K,h,w) fp32 or NULL      — if non-NULL, predict = argmax over the K planes
 *   predict  (B,h,w) int64 or NULL       — used when seg is NULL
 * ----------------------------------------------------------------------------------------------*/
int pcl_class_stats(const pcl_geom* g, const int64_t* labels, const float* seg, const int64_t* predict,
                    uint16_t* keys, int32_t* chunk_pref, int32_t* counts, void* stream);

/* a4: class filter (count > max_views), TC, V = min(max_samples / TC, max_views), hard/easy split
 * rule and the class-sorted anchor row layout.  Replaces lib/loss/loss_contrast.py:37-48,63-77.
 * Reads the per-image key totals `counts` written by pcl_class_stats; writes the plan. */
int pcl_plan_anchors(const pcl_geom* g, const int32_t* counts, int32_t* plan, void* stream);

/* a4 (second half) + gather: choose the pixels of every anchor row and gather their embeddings.
 * Replaces lib/loss/loss_contrast.py:79-86 (randperm, index, X_[ptr] = X[ii, indices]) and the
 * 268 MB permute+contiguous of :141-142 (never materialised here).
 *   ranks     NULL -> device RNG (keyed Feistel permutation, `seed`), no host round trip;
 *             else (TC,V) int32 table: ranks[t*V+v] = perm value used for view v of pair t
 *             (hard ranks first, then easy ranks) — replay of the reference's torch.randperm draws.
 *   normalize 0: embed is already L2-normalised (projection.py:24 ran upstream);
 *             1: embed is the raw projection, only the gathered columns are normalised here.
 * Outputs (row s = class-sorted anchor index, rows >= A are zero-filled):
 *   anchor_meta (4,max_samples) int32: pixel, image, class, reference row r = v*TC + t
 *   anchors_f32 (max_samples,D), anchors_bf16 (max_samples rounded up to 128, D) or NULL,
 *   inv_norm (max_samples) fp32 (1/||x|| of the raw column; 1 when normalize == 0),
 *   norm_max  optional (may be NULL): 1 float, max over anchors of ||a||. */
int pcl_select_gather(const pcl_geom* g, const float* embed, const uint16_t* keys, const int32_t* chunk_pref,
                      const int32_t* plan, const int32_t* ranks, uint64_t seed, int normalize,
                      int32_t* anchor_meta, float* anchors_f32, void* anchors_bf16, float* inv_norm,
                      float* norm_max, void* stream);

/* ------------------------------------------------------------------------------------------------
 * a5 + a6: the contrast set and the InfoNCE sweep.
 * Replaces lib/loss/loss_contrast.py:91-128 and lib/loss/loss_contrast_mem.py:91-152.
 * ----------------------------------------------------------------------------------------------*/
typedef struct {
  /* anchors (rows); device scalar plan[PCL_PLAN_A] gives the live row count, a_rows its upper bound */
  const float*   anchors;        /* (a_rows, D) fp32, class-sorted                                   */
  const int32_t* anchor_cls;     /* (a_rows) int32                                                   */
  const int32_t* diag_col;       /* (a_rows) int32 contrast column removed from the positives (Q1)   */
  const int32_t* plan;           /* plan buffer or NULL (then a_live = a_rows)                       */
  int32_t a_rows;
  int32_t D;
  /* contrast set.  mode 0: self-contrast (columns == anchors, loss_contrast.py:91-128)
   *                mode 1: memory bank, read in place from the two queues (mem:91-105,221):
   *                        column n = (c-1)*R + q, R = M0+M1, c = 1..K-1 (class 0 skipped, Q2), q < M0 -> segment
   *                        row, else pixel row; plus `R` all-zero columns of label 0 handled analytically (Q3)
   *                mode 2: explicit matrix `contrast` (n_cols, D) with labels `contrast_cls`           */
  int32_t mode;
  const float*   segment_queue;  /* (K, M0, D) fp32                                                  */
  const float*   pixel_queue;    /* (K, M1, D) fp32, or NULL with bank_M1 == 0 (pre-concatenated queue
                                    (K, R, D) passed as segment_queue with bank_M0 == R)             */
  int32_t bank_K, bank_M0, bank_M1;
  const float*   contrast;       /* mode 2                                                           */
  const int32_t* contrast_cls;   /* mode 2                                                           */
  int32_t n_cols;                /* mode 2                                                           */
  float temperature, base_temperature;
  int32_t nan_safe;              /* 0: rows without positives give NaN like the reference (Q8); 1: they give 0 */
} pcl_sweep_desc;

typedef struct {
  int64_t n_real_cols;         /* streamed columns                                                  */
  int32_t row_tiles, splits;   /* launch grid of the SIMT sweep                                     */
  int64_t partial_f32;         /* splits * a_rows_padded floats, per partial statistic (5 of them)  */
  int64_t rowstat_f32;         /* a_rows floats, per final statistic (6: m, neg, possum, s, npos, row_loss) */
  int64_t dpartial_f32;        /* splits * a_rows_padded * D floats (backward partial dA)           */
} pcl_sweep_sizes_t;

int pcl_sweep_sizes(const pcl_sweep_desc* d, pcl_sweep_sizes_t* out);

/* Forward: loss (1 float) and per-row statistics.  partials: 5 * partial_f32 floats of scratch;
 * rowstats: 6 * rowstat_f32 floats (m, neg, possum, s, npos, row_loss), kept for the backward. */
int pcl_infonce_fwd(const pcl_sweep_desc* d, float* partials, float* rowstats, float* loss, void* stream);

/* Backward: dA (a_rows, D) = d loss / d anchors (closed form, SURVEY appendix A), multiplied by the
 * upstream gradient *grad_loss (device scalar, may be NULL = 1).  dpartials: scratch. */
int pcl_infonce_bwd(const pcl_sweep_desc* d, const float* rowstats, const float* grad_loss, float* dpartials,
                    float* dA, void* stream);

/* ------------------------------------------------------------------------------------------------
 * a10 (SURVEY §8): per-anchor top-k hard-negative selection on the exact fp32 sweep — an extension the
 * reference code does not have (lib/loss/loss_contrast.py:116-117 and loss_contrast_mem.py:140-141 sum ALL
 * negatives), default off.  Neg_i = sum of exp(l - m_i) over the k negatives of anchor i with the largest
 * logits; ties at the k-th value share the remaining slots equally (order independent); rows with <= k
 * negatives keep all of them (== pcl_infonce_fwd).  Exact 3-level radix select on the fp32 logits, streamed:
 * three histogram sweeps + the weighted NEG sweep + the stock POS sweep; the A x N logits are never stored.
 *   scratch  uint32 words, pcl_topk_scratch_u32(d) of them (negative = pcl_status): per-row radix bins followed by
 *            the selection result sel[4][a_rows] = tau key (order-preserving integer image of the k-th largest
 *            negative logit; 0 = all kept), tie weight (float bits), G = #negatives above tau, E = #ties at tau.
 *            The SAME scratch must be passed to the backward.
 *   partials / rowstats / loss / dpartials / dA: as pcl_infonce_fwd / pcl_infonce_bwd.
 * ----------------------------------------------------------------------------------------------*/
int64_t pcl_topk_scratch_u32(const pcl_sweep_desc* d);
int pcl_infonce_topk_fwd(const pcl_sweep_desc* d, int32_t k, uint32_t* scratch, float* partials, float* rowstats,
                         float* loss, void* stream);
int pcl_infonce_topk_bwd(const pcl_sweep_desc* d, int32_t k, uint32_t* scratch, const float* rowstats,
                         const float* grad_loss, float* dpartials, float* dA, void* stream);

/* dA -> dense NCHW gradient of the embedding (zero fill + scatter; with normalize == 1 the
 * projection-normalise backward of the touched columns is fused in: dx = (g - y (y.g)) / ||x||).
 * Replaces the autograd backward of loss_contrast.py:83-85,:141-142 (152 SelectBackward0 zero fills). */
int pcl_scatter_grad(const pcl_geom* g, const int32_t* plan, const int32_t* anchor_meta, const float* dA,
                     const float* anchors_f32, const float* inv_norm, int normalize, float* grad_embed,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * a1: projection-head normalise, lib/models/modules/projection.py:24  (F.normalize(x, p=2, dim=1)).
 * ----------------------------------------------------------------------------------------------*/
int pcl_l2norm_fwd(const float* x, float* y, int32_t B, int32_t D, int64_t HW, void* stream);
int pcl_l2norm_bwd(const float* x, const float* gy, float* gx, int32_t B, int32_t D, int64_t HW, void* stream);

/* ------------------------------------------------------------------------------------------------
 * §8f row 2: the projection head's last 1x1 convolution and its L2 normalise as one bf16 wgmma GEMM (fp32 accumulate),
 * forward and backward.  Replaces lib/models/modules/projection.py:17-24 (the final nn.Conv2d(Cin, 256, 1) of the
 * head, then F.normalize(p=2, dim=1)) and their autograd backward.  Output channels are fixed at 256.
 *   x (B,Cin,HW) fp32 NCHW, weight (256,Cin) fp32, bias (256) fp32 or NULL, zn (B,256,HW) fp32, inv_norm (B*HW) fp32
 *   (1 / max(|z|, 1e-12) per pixel; kept for the backward).
 *   wpack    pcl_proj_workspace_bytes(B, Cin, HW, 0) bytes: bf16 copies of the weight written by pcl_proj_pack; pack
 *            again whenever the weight changes.  Used by the forward and the backward.
 *   scratch  pcl_proj_workspace_bytes(B, Cin, HW, 1) bytes: backward-only (bf16 gz, split-K weight-gradient partials).
 *   pcl_proj_bwd writes gx (B,Cin,HW), gw (256,Cin) and gb (256, may be NULL); gw and gb are reduced in a fixed order
 *   (bit-reproducible).  The size query returns a negative pcl_status for an unsupported shape.
 * ----------------------------------------------------------------------------------------------*/
int64_t pcl_proj_workspace_bytes(int32_t B, int32_t Cin, int64_t HW, int32_t which);
int pcl_proj_pack(const float* weight, int32_t Cin, void* wpack, void* stream);
int pcl_proj_fwd(const float* x, const void* wpack, const float* bias, int32_t B, int32_t Cin, int64_t HW, float* zn,
                 float* inv_norm, void* stream);
int pcl_proj_bwd(const float* x, const float* zn, const float* inv_norm, const float* gzn, const void* wpack, int32_t B,
                 int32_t Cin, int64_t HW, void* scratch, float* gx, float* gw, float* gb, void* stream);

/* The two calls above with the activations x, zn, gzn and gx of element type `dtype`: PCL_DT_F32 (exactly the calls
 * above) or PCL_DT_BF16; any other code, PCL_DT_F16 included, returns PCL_ERR_ARG (an fp16 activation would be rounded
 * to the bf16 GEMM operand).  bf16 activations are converted to fp32 on load (exact) and everything is computed as for
 * fp32 activations, so against the fp32 call on the converted inputs: zn and gx are its zn and gx rounded to
 * nearest-even, inv_norm, gw and gb are bit-identical.  inv_norm, weight, bias, gw and gb stay fp32; wpack and scratch
 * are sized and packed as above. */
int pcl_proj_fwd_dt(const void* x, int32_t dtype, const void* wpack, const float* bias, int32_t B, int32_t Cin,
                    int64_t HW, void* zn, float* inv_norm, void* stream);
int pcl_proj_bwd_dt(const void* x, int32_t dtype, const void* zn, const float* inv_norm, const void* gzn,
                    const void* wpack, int32_t B, int32_t Cin, int64_t HW, void* scratch, void* gx, float* gw,
                    float* gb, void* stream);

/* The head's BatchNorm2d / SyncBatchNorm and ReLU fused into the calls above: zn = normalize(conv(relu(bn(y)))) with
 * y (B,Cin,HW) of element type `dtype` (PCL_DT_F32 or PCL_DT_BF16; anything else returns PCL_ERR_ARG).  Training:
 *   pcl_proj_bn_stats_dt     sums (2*Cin + 1 doubles): sum y, sum y^2 per channel, then the count B*HW.  fp64 and
 *                            bit-reproducible; sums of several ranks add up (SyncBatchNorm all-reduces them).
 *   pcl_proj_bn_finalize     training 1: batch mean / biased variance from sums; running_mean / running_var updated
 *                            in place (momentum, unbiased variance over the count); training 0: the running buffers,
 *                            nothing updated, sums may be NULL.  Writes bn_state (pcl_proj_bn_workspace_bytes(.., 0) bytes,
 *                            16-byte aligned).
 *   pcl_proj_bn_fwd_dt       pcl_proj_fwd_dt on max(0, (y - mean) invstd gamma + beta), never materialised.
 *   pcl_proj_bn_bwd_dt       pcl_proj_bwd_dt through the ReLU: gu = the gradient of the BN output (B,Cin,HW, dtype),
 *                            gw, gb as above; gsum (2*Cin floats) = sum gu, sum gu x_hat per channel; gbeta, ggamma
 *                            (may be NULL) the same local sums.  scratch: pcl_proj_bn_workspace_bytes(.., 1) bytes.
 *   pcl_proj_bn_input_grad_dt  gu -> the gradient of y, in place in g.  training 1 uses gsum (summed over ranks for
 *                            SyncBatchNorm) and the count of the statistics; training 0: gamma invstd gu.
 * No call synchronises with the host. */
int64_t pcl_proj_bn_workspace_bytes(int32_t B, int32_t Cin, int64_t HW, int32_t which);
int pcl_proj_bn_stats_dt(const void* y, int32_t dtype, int32_t B, int32_t Cin, int64_t HW, double* sums, void* stream);
int pcl_proj_bn_finalize(const double* sums, const float* gamma, const float* beta, float* running_mean,
                         float* running_var, int32_t Cin, float eps, float momentum, int32_t training, void* bn_state,
                         void* stream);
int pcl_proj_bn_fwd_dt(const void* y, int32_t dtype, const void* bn_state, const void* wpack, const float* bias,
                       int32_t B, int32_t Cin, int64_t HW, void* zn, float* inv_norm, void* stream);
int pcl_proj_bn_bwd_dt(const void* y, int32_t dtype, const void* bn_state, const void* zn, const float* inv_norm,
                       const void* gzn, const void* wpack, int32_t B, int32_t Cin, int64_t HW, void* scratch, void* gu,
                       float* gw, float* gb, float* gsum, float* ggamma, float* gbeta, void* stream);
int pcl_proj_bn_input_grad_dt(const void* y, int32_t dtype, const void* bn_state, const float* gsum, int32_t B,
                              int32_t Cin, int64_t HW, int32_t training, void* g, void* stream);

/* The backward of the calls above when gzn is zero outside n_cols anchor columns (what pcl_step_backward_cols hands
 * over): cols (n_cols, 256) fp32, col_pix[a] = b*HW + p, or < 0 for an unused column.  Replaces pcl_proj_bn_bwd_dt +
 * pcl_proj_bn_input_grad_dt (csrc/pcl_norm.cu:1347, :1371) on the dense gzn built from the columns; no dense gzn, bf16
 * gz or dense gu is written, and the last conv's GEMMs run over the columns only.  ReLU' and the BN backward of a
 * gradient that is zero off the anchors leave g_y = gamma invstd (gu - sum gu / n - x_hat sum(gu x_hat) / n): the
 * anchors' gu plus a per-channel affine function of x_hat.  Plain fp32 on w2, the fp32 (256, Cin) weight of the last
 * conv; every sum runs in a fixed order (bit-reproducible).
 *   pcl_proj_bn_cols_workspace_bytes  scratch bytes for (n_cols, Cin).
 *   pcl_proj_bn_bwd_cols_dt       gw (256, Cin), gb (may be NULL), gsum (2*Cin) and gbeta / ggamma (may be NULL) as
 *                                 pcl_proj_bn_bwd_dt defines them; the anchors' gu stay in scratch for the next call.
 *   pcl_proj_bn_input_grad_cols_dt  writes the whole gradient g of y (B,Cin,HW, dtype) from y, bn_state, gsum (summed
 *                                 over ranks for SyncBatchNorm) and the scratch of the call above; training 0 gives
 *                                 gamma invstd gu at the anchors and 0 elsewhere.
 * y, zn and g have element type `dtype` (PCL_DT_F32 or PCL_DT_BF16).  No call synchronises with the host. */
int64_t pcl_proj_bn_cols_workspace_bytes(int32_t n_cols, int32_t Cin);
int pcl_proj_bn_bwd_cols_dt(const void* y, int32_t dtype, const void* bn_state, const void* zn, const float* inv_norm,
                            const float* cols, const int32_t* col_pix, int32_t n_cols, const float* w2, int32_t B,
                            int32_t Cin, int64_t HW, void* scratch, float* gw, float* gb, float* gsum, float* ggamma,
                            float* gbeta, void* stream);
int pcl_proj_bn_input_grad_cols_dt(const void* y, int32_t dtype, const void* bn_state, const float* gsum,
                                   const void* scratch, const int32_t* col_pix, int32_t n_cols, int32_t B, int32_t Cin,
                                   int64_t HW, int32_t training, void* g, void* stream);

/* The head's first 1x1 convolution (Conv2d(C, C, 1), lib/models/modules/projection.py:17-19) in front of the calls
 * above, as bf16 wgmma GEMMs (fp32 accumulate), forward and backward, with the BatchNorm statistics of its output in the
 * forward's epilogue.  x, y, gy and gx (B,C,HW) have element type `dtype` (PCL_DT_F32 or PCL_DT_BF16; anything else
 * returns PCL_ERR_ARG); an fp32 x is rounded to bf16 to nearest-even, a bf16 x is the operand as it is.  w1 (C,C),
 * b1 (C), gw1 (C,C) and gb1 (C) are fp32.  Any C >= 1 and any HW.
 *   pack     pcl_proj_conv1_workspace_bytes(B, C, HW, 0) bytes: the bf16 copies of w1 written by pcl_proj_conv1_pack;
 *            pack again whenever w1 changes.  Used by the forward and the backward.
 *   pcl_proj_conv1_fwd_dt  y = w1 x + b1 per pixel (b1 may be NULL), stored in `dtype`.  sums (may be NULL: no
 *            statistics) gets exactly what pcl_proj_bn_stats_dt(y, ...) writes: the fp64 sums of the stored y and y^2
 *            per channel, then the count B*HW, in a fixed order (bit-reproducible).  scratch (may be NULL when sums
 *            is): pcl_proj_conv1_workspace_bytes(.., 1) bytes.
 *   pcl_proj_conv1_bwd_dt  gx = w1^T gy per pixel (gx may be NULL: not computed), gw1 = sum over pixels of gy x^T and
 *            gb1 (may be NULL) = sum over pixels of gy, gy rounded to bf16 for the GEMMs; gw1 and gb1 are reduced in a
 *            fixed order (bit-reproducible).  scratch: pcl_proj_conv1_workspace_bytes(.., 2) bytes.
 * The size query returns a negative pcl_status for an unsupported shape.  No call synchronises with the host. */
int64_t pcl_proj_conv1_workspace_bytes(int32_t B, int32_t C, int64_t HW, int32_t which);
int pcl_proj_conv1_pack(const float* w1, int32_t C, void* pack, void* stream);
int pcl_proj_conv1_fwd_dt(const void* x, int32_t dtype, const void* pack, const float* b1, int32_t B, int32_t C,
                          int64_t HW, void* y, double* sums, void* scratch, void* stream);
int pcl_proj_conv1_bwd_dt(const void* x, int32_t dtype, const void* gy, const void* pack, int32_t B, int32_t C,
                          int64_t HW, void* scratch, void* gx, float* gw1, float* gb1, void* stream);

/* ------------------------------------------------------------------------------------------------
 * §8f row 1 (next row): the segmentation CE of ContrastCELoss.forward, fused.  Replaces
 * lib/loss/loss_contrast.py:180-181 (F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True)) +
 * lib/loss/loss_helper.py:169-212 (nn.CrossEntropyLoss(weight, ignore_index, reduction mean)) and their autograd
 * backward; the (B,K,Himg,Wimg) up-sampled logits are never materialised.
 *   seg (B,K,h,w) fp32, target (B,Himg,Wimg) int64, class_weight (K) fp32 or NULL, scratch: pcl_seg_ce_scratch_floats.
 * ----------------------------------------------------------------------------------------------*/
int64_t pcl_seg_ce_scratch_floats(int32_t B, int32_t Himg, int32_t Wimg);
int pcl_seg_ce_fwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K, int32_t h,
                   int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index, float* scratch, float* loss, void* stream);
int pcl_seg_ce_bwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K, int32_t h,
                   int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index, const float* scratch,
                   const float* grad_loss, float* dseg, void* stream);
/* The same forward and backward in one call, for a terminal loss whose upstream gradient is a device scalar that exists
 * when the call runs (a captured criterion): replaces the same lines (loss_contrast.py:180-181 + loss_helper.py:169-212
 * and their autograd backward).  With K <= 24 (one class chunk of the backward tile) it is one tile pass that keeps no
 * per-pixel log-sum-exp between forward and backward, stages the logit patch once and reads the labels once; with more
 * classes it runs the kernels of pcl_seg_ce_fwd and pcl_seg_ce_bwd.  loss (1 float) is pcl_seg_ce_fwd's to the bit;
 * dseg = grad_scale[0] (1 when NULL) * d loss / d seg, pcl_seg_ce_bwd's to the last ulp or two (fp32 atomics in both).
 * Every pixel ignored: loss NaN, dseg zero.  A label grid smaller than the logits (Himg < h or Wimg < w):
 * PCL_ERR_UNSUPPORTED.  scratch: pcl_seg_ce_fwd_bwd_scratch_floats floats. */
int64_t pcl_seg_ce_fwd_bwd_scratch_floats(int32_t B, int32_t K, int32_t Himg, int32_t Wimg);
int pcl_seg_ce_fwd_bwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K,
                       int32_t h, int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index, float* scratch,
                       const float* grad_scale, float* loss, float* dseg, void* stream);

/* ------------------------------------------------------------------------------------------------
 * §8f row f5: the RMI segmentation loss of the contrast wrappers with contrast.use_rmi, fused.  Replaces
 * F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True) + RMILoss.forward (sigmoid path:
 * lib/loss/rmi_loss.py:200-402, via FSRMILoss / FSAuxRMILoss, lib/loss/loss_helper.py:316-369) and its autograd
 * backward; neither the (B,K,Himg,Wimg) logits / one-hot / probabilities nor the float64 neighbour vectors are
 * materialised.  num_classes = K; a label < 0 counts as 255, a pixel is valid when its label < K (target is read only).
 *   seg (B,K,h,w) fp32 with Himg >= h, Wimg >= w; target (B,Himg,Wimg) int64; radius 1-4; pool_way 0 (max) or 1 (avg);
 *   pool_stride (== pool size) 1-4; lambda_way != 0: loss_weight * (lambda * bce + (1 - lambda) * rmi), else
 *   loss_weight * (bce + lambda * rmi).  Radius 5-10, pool way 2, down-sampling, more than 256 classes or a pooled map
 *   smaller than the radius return PCL_ERR_UNSUPPORTED.
 *   scratch: pcl_rmi_scratch_bytes (host only; a negative PCL_ERR_* for a refused request).  pcl_rmi_bwd reads the
 *   scratch its pcl_rmi_fwd wrote.  The loss is bit-reproducible; dseg to the last ulp or two (fp32 atomics).
 * ----------------------------------------------------------------------------------------------*/
int64_t pcl_rmi_scratch_bytes(int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg, int32_t Wimg, int32_t radius,
                              int32_t pool_way, int32_t pool_stride);
int pcl_rmi_fwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg,
                int32_t Wimg, int32_t radius, int32_t pool_way, int32_t pool_stride, float weight_lambda,
                int32_t lambda_way, float loss_weight, void* scratch, float* loss, void* stream);
int pcl_rmi_bwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg,
                int32_t Wimg, int32_t radius, int32_t pool_way, int32_t pool_stride, float weight_lambda,
                int32_t lambda_way, float loss_weight, void* scratch, const float* grad_loss, float* dseg, void* stream);

/* ------------------------------------------------------------------------------------------------
 * §8f row f6: the Lovasz-softmax term of FSCELOVASZLoss (lib/loss/loss_helper.py:77-124, selected by
 * contrast.use_lovasz in lib/loss/loss_contrast_mem.py:187-194), fused.  Replaces F.interpolate(seg, (Himg,Wimg),
 * bilinear, align_corners=True) + softmax + lovasz_softmax_flat(*flatten_probas(...), only_present=True)
 * (lib/loss/lovasz_loss.py:216-267) and its autograd backward; the (B,K,Himg,Wimg) logits and probabilities are never
 * materialised and no call syncs with the host (capturable).
 *   seg (B,K,h,w) fp32 with Himg >= h, Wimg >= w; target (B,Himg,Wimg) int64 (read only).  A pixel counts when its label
 *   is not ignore_index and lies in [0, K); the others are ignored (the reference's CE raises on them).  Pixels are
 *   pooled over the whole batch; the loss is the mean over the classes present among them, 0 (zero gradient) when none.
 *   Equal errors are ordered by ascending pixel index (b*Himg + y)*Wimg + x, i.e. a stable descending sort; the loss
 *   does not depend on that order, the per-pixel gradient does.  p exactly 0 or 1 gets a zero gradient (abs').
 *   A label grid smaller than seg, K > 256 or B*Himg*Wimg >= 2^31 return PCL_ERR_UNSUPPORTED.
 *   scratch: pcl_lovasz_scratch_bytes (host only; a negative PCL_ERR_* for a refused request).  pcl_lovasz_bwd reads the
 *   scratch its pcl_lovasz_fwd wrote.  The loss is bit-reproducible; dseg to the last ulp or two (fp32 atomics).
 * ----------------------------------------------------------------------------------------------*/
int64_t pcl_lovasz_scratch_bytes(int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg, int32_t Wimg);
int pcl_lovasz_fwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg,
                   int32_t Wimg, int32_t ignore_index, void* scratch, float* loss, void* stream);
int pcl_lovasz_bwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg,
                   int32_t Wimg, int32_t ignore_index, void* scratch, const float* grad_loss, float* dseg, void* stream);

/* ------------------------------------------------------------------------------------------------
 * §8f row f7: the OHEM cross-entropy of FSOhemCELoss and of the seg term of FSAuxOhemCELoss
 * (lib/loss/loss_helper.py:215-261), fused.  Replaces F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True) +
 * softmax + gather of the target probability + sort of the labelled pixels + CrossEntropyLoss(weight,
 * reduction='none') + the selection, and its autograd backward; the (B,K,Himg,Wimg) logits and probabilities are never
 * materialised and no call syncs with the host (capturable).
 *   seg (B,K,h,w) fp32 with Himg >= h, Wimg >= w; target (B,Himg,Wimg) int64 (read only); class_weight (K) fp32 or NULL.
 *   A pixel counts when its label is not ignore_index and lies in [0, K); the others are ignored (the reference raises
 *   on labels outside [0, K)).  Over the n counted pixels of the whole batch, p_t = softmax(up(seg))[t]:
 *     kth = the m-th smallest p_t, 0-based, m = min(min_kept, n - 1)   (min_kept >= 1: the module passes
 *           max(1, ohem_minkeep));
 *     threshold = max(kth, thresh), compared in fp32 (thresh is passed as a float, as torch compares it);
 *     the selected pixels are those with p_t < threshold (strict: pixels tied at the threshold are all left out);
 *     loss_i = w[t_i] * nll_i; reduction 0 ('mean' / 'elementwise_mean'): sum(loss_i) / count (not divided by the
 *     sum of the weights); reduction 1 ('sum'): the plain sum.  Any other reduction is PCL_ERR_ARG.
 *   The selection carries no gradient: a selected pixel's gradient is s * w_t * (softmax - onehot_t), s = grad / count
 *   ('mean') or grad ('sum').  No counted pixel (n = 0): the loss is 0 with a zero gradient (the reference raises on the
 *   empty sort).  n > 0 with an empty selection (e.g. n = 1, or every p_t equal): NaN for 'mean', 0 for 'sum', with a
 *   zero gradient, as in the reference.
 *   A label grid smaller than seg, K > 256 or B*Himg*Wimg >= 2^31 return PCL_ERR_UNSUPPORTED.
 *   scratch: pcl_ohem_ce_scratch_bytes (host only; a negative PCL_ERR_* for a refused request), 256-byte aligned.  After
 *   pcl_ohem_ce_fwd its first 32 bytes hold float loss, float denominator, float threshold, int32 select (1 when the
 *   exact select ran, 0 when fp32(thresh) decided), int32 n, int32 count(p_t < thresh), int32 selected count; from byte
 *   256 on the B*Himg*Wimg floats p_t in (b, y, x) order, NaN at the pixels that do not count.
 *   pcl_ohem_ce_bwd reads the scratch its pcl_ohem_ce_fwd wrote.  The loss is bit-reproducible; dseg to the last ulp or
 *   two (fp32 atomics).
 * ----------------------------------------------------------------------------------------------*/
int64_t pcl_ohem_ce_scratch_bytes(int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg, int32_t Wimg);
int pcl_ohem_ce_fwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K, int32_t h,
                    int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index, float thresh, int64_t min_kept,
                    int32_t reduction, void* scratch, float* loss, void* stream);
int pcl_ohem_ce_bwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K, int32_t h,
                    int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index, const void* scratch,
                    const float* grad_loss, float* dseg, void* stream);

/* ------------------------------------------------------------------------------------------------
 * a7 + a8: memory bank.  Replaces segmentor/trainer_contrastive.py:102-138 (_dequeue_and_enqueue).
 * Step 1 (parallel): build this rank's enqueue packet.  Step 2 (ordered): apply the packets of all
 * ranks in rank order — world 1 reproduces the reference exactly, world > 1 is the allgather merge
 * (SURVEY §8e).  Packet layout per (image b, class c) slot, slot = b*K + c, `slot_f32` floats:
 *   [0] n pixels of the class in the sub-sampled label map (0 = slot empty)   [1] K' = min(n, F)
 *   [2 .. 2+D)            normalised segment mean          (trainer_contrastive.py:120-122)
 *   [2+D .. 2+D+F*D)      K' normalised pixel rows         (trainer_contrastive.py:126-130)
 * ----------------------------------------------------------------------------------------------*/
typedef struct {
  int32_t B, D, h, w;          /* keys (B,D,h,w) fp32                                               */
  int32_t Himg, Wimg;          /* labels (B,Himg,Wimg) int64                                        */
  int32_t K, M;                /* queues (K,M,D)                                                    */
  int32_t network_stride;      /* labels[:, ::s, ::s]  (Q6: flat index of that grid == feature column) */
  int32_t pixel_update_freq;   /* F                                                                 */
} pcl_bank_geom;

int64_t pcl_bank_packet_floats(const pcl_bank_geom* g);    /* floats in one rank's packet           */
int64_t pcl_bank_scratch_floats(const pcl_bank_geom* g);   /* floats of scratch for pcl_bank_packet */

/* ranks: NULL -> device RNG with `seed`; else (B*K, F) int32 table of perm values per slot. */
int pcl_bank_packet(const pcl_bank_geom* g, const float* keys, const int64_t* labels, const int32_t* ranks,
                    uint64_t seed, float* scratch, float* packet, void* stream);

/* Same for a captured launch sequence (CUDA graph): kernel arguments are frozen at capture, so the per-call part of the
 * seed is read from device memory: effective seed = seed + *seed_offset (uint64 on the device, e.g. the step counter
 * pcl_step_ranks advances; NULL -> 0).  Device RNG only. */
int pcl_bank_packet_dev(const pcl_bank_geom* g, const float* keys, const int64_t* labels, uint64_t seed,
                        const uint64_t* seed_offset, float* scratch, float* packet, void* stream);

/* The two calls above for keys of element type keys_dtype (PCL_DT_*; bf16 / fp16 keys are converted on load, the
 * packet is fp32 and bit-identical to the one built from the keys converted to fp32). */
int pcl_bank_packet_dt(const pcl_bank_geom* g, const void* keys, int32_t keys_dtype, const int64_t* labels,
                       const int32_t* ranks, uint64_t seed, float* scratch, float* packet, void* stream);
int pcl_bank_packet_dev_dt(const pcl_bank_geom* g, const void* keys, int32_t keys_dtype, const int64_t* labels,
                           uint64_t seed, const uint64_t* seed_offset, float* scratch, float* packet, void* stream);

/* Apply `world` packets (contiguous, rank-major) to the queues in place, with the result of the reference's sequential
 * per-image loop over the gathered batch (trainer_contrastive.py:96-139): every queue row is written once, by the LAST
 * of the world * B slots that would have written it.  world * B <= 1024 (PCL_ERR_UNSUPPORTED otherwise).
 * shadow_bf16 (optional, ((K-1)*2M rounded up to 256, D) bf16) is the engine's class-blocked bf16 copy used by the
 * tensor path. */
int pcl_bank_apply(const pcl_bank_geom* g, const float* packets, int32_t world, float* segment_queue,
                   int64_t* segment_queue_ptr, float* pixel_queue, int64_t* pixel_queue_ptr,
                   void* shadow_bf16, void* stream);

/* Same; additionally advances *enqueue_counter (device uint64, may be NULL) when done: the seed offset of the NEXT
 * pcl_bank_packet_dev of a captured sequence. */
int pcl_bank_apply_ctr(const pcl_bank_geom* g, const float* packets, int32_t world, float* segment_queue,
                       int64_t* segment_queue_ptr, float* pixel_queue, int64_t* pixel_queue_ptr,
                       void* shadow_bf16, uint64_t* enqueue_counter, void* stream);

/* Rebuild the bf16 shadow from the fp32 queues (after a checkpoint load / external write). */
int pcl_bank_shadow_rebuild(const float* segment_queue, const float* pixel_queue, int32_t K, int32_t M,
                            int32_t D, void* shadow_bf16, void* stream);

/* ------------------------------------------------------------------------------------------------
 * a6 on the tensor cores (wgmma + TMA, bf16 operands, fp32 accumulate), D must be 256.
 * Same semantics and row-statistic layout as pcl_infonce_fwd; operands are bf16 copies:
 *   anchors_bf16   (a_rows rounded up to 128, 256) bf16 — written here from anchors_f32 when that is non-NULL
 *   contrast_bf16  mode 1: the bank shadow ((K-1)*R rounded up to 256 rows, class-blocked, see pcl_bank_apply);
 *                  mode 2: (contrast_rows_alloc, 256) rows with labels contrast_cls (sorted = labels are
 *                  non-decreasing, enables the no-compare fast path); mode 0: ignored (columns == anchors)
 *   contrast_norm_bound  upper bound of the contrast rows' L2 norm (1 for a normalised bank); only has to keep
 *                  exp() in range — the loss does not depend on it
 * ----------------------------------------------------------------------------------------------*/
typedef struct {
  const float*   anchors_f32;    /* (a_rows, 256) or NULL when anchors_bf16 is already filled                */
  void*          anchors_bf16;
  const int32_t* anchor_cls; const int32_t* diag_col; const int32_t* plan;
  int32_t a_rows, D;
  int32_t mode;
  const void*    contrast_bf16;
  const int32_t* contrast_cls;
  int64_t n_cols; int64_t contrast_rows_alloc;
  int32_t bank_K, bank_R, sorted;
  float contrast_norm_bound;
  float temperature, base_temperature;
  int32_t nan_safe;
  int32_t neg_only;              /* 1: stop after the similarity + negative-sum sweep (the dense contraction alone,
                                    used to report its roofline fraction); loss / rowstats are then not final */
} pcl_tc_desc;

int pcl_tc_sizes(const pcl_tc_desc* d, pcl_sweep_sizes_t* out);
/* a10 on the tensor path (same semantics as pcl_infonce_topk_fwd/bwd, selection on the fp32-accumulated logits of the bf16
 * operands): scratch = pcl_tc_topk_scratch_u32(d) uint32 (per-row radix bins + the selection state, kept for the
 * backward); three extra similarity sweeps whose epilogue bins the logit keys (red.global), then the weighted sweep. */
int64_t pcl_tc_topk_scratch_u32(const pcl_tc_desc* d);
int pcl_infonce_tc_topk_fwd(const pcl_tc_desc* d, int32_t k, uint32_t* scratch, float* row_m2, float* partials,
                            float* rowstats, float* loss, void* stream);
int pcl_infonce_tc_topk_bwd(const pcl_tc_desc* d, int32_t k, const uint32_t* scratch, const float* row_m2,
                            const float* rowstats, const float* grad_loss, float* dpartials, float* dA, void* stream);
int pcl_to_bf16(const float* src, void* dst_bf16, int64_t n_real, int64_t n_total, void* stream);
/* row_m2: (a_rows rounded up to 256) + 512 floats of scratch (per-row stabiliser, kept for the backward,
 * followed by the per-label column bounds of a sorted explicit contrast set). */
int pcl_infonce_tc_fwd(const pcl_tc_desc* d, float* row_m2, float* partials, float* rowstats, float* loss,
                       void* stream);
/* Backward on the tensor cores: dA (a_rows, 256) fp32 = d loss / d anchors * (*grad_loss or 1).  row_m2 and rowstats
 * come from pcl_infonce_tc_fwd; dpartials: pcl_tc_sizes().dpartial_f32 floats of scratch. */
int pcl_infonce_tc_bwd(const pcl_tc_desc* d, const float* row_m2, const float* rowstats, const float* grad_loss,
                       float* dpartials, float* dA, void* stream);
/* Pipeline self-test: raw similarity tiles S = A.C^T into dump[(a_rows up to 256) x (n_cols up to 256)] fp32. */
int pcl_tc_dump_logits(const pcl_tc_desc* d, float* row_m2, float* dump, void* stream);

/* ------------------------------------------------------------------------------------------------
 * One loss step = the calls above chained on one stream behind a single descriptor (what
 * PixelContrastLoss.forward / its autograd backward bind; lib/loss/loss_contrast.py:130-147,
 * lib/loss/loss_contrast_mem.py:154-171).  All scratch is caller-owned.
 * ----------------------------------------------------------------------------------------------*/
typedef struct {
  pcl_geom g;
  /* inputs */
  const float*   embed;          /* (B,D,h,w)                                                        */
  const int64_t* labels;         /* (B,Himg,Wimg)                                                    */
  const float*   seg;            /* (B,K,h,w) or NULL                                                */
  const int64_t* predict;        /* (B,h,w) or NULL                                                  */
  const int32_t* ranks;          /* injected permutation values or NULL (device RNG)                 */
  uint64_t seed;
  int32_t normalize;
  /* contrast set: mode 0 self, 1 bank */
  int32_t mode;
  const float* segment_queue; const float* pixel_queue;
  int32_t bank_K, bank_M0, bank_M1;
  float temperature, base_temperature;
  int32_t nan_safe;
  /* scratch */
  uint16_t* keys; int32_t* chunk_pref; int32_t* counts; int32_t* plan; int32_t* anchor_meta;
  float* anchors_f32; void* anchors_bf16; float* inv_norm; float* norm_max;
  float* partials; float* rowstats; float* dpartials; float* dA;
  /* sweep selection: 0 = exact fp32 SIMT sweep (any D % 32 == 0, D <= 256); 1 = bf16 wgmma sweep (D == 256).
   * The tensor path reads the bank through its bf16 shadow (pcl_bank_apply / pcl_bank_shadow_rebuild). */
  int32_t precision;
  const void* shadow_bf16; int64_t shadow_rows;
  float contrast_norm_bound;
  float* row_m2;                 /* (max_samples rounded up to 256) + 512 floats (tensor path only)  */
  /* outputs */
  float* loss;                   /* 1 float                                                          */
  float* grad_embed;             /* (B,D,h,w), written by pcl_step_backward                          */
  uint32_t* sync;                /* optional: 1024 words of device memory, ZERO before the first call, owned by this step:
                                  * inter-CTA counters of the fused kernels (re-armed by the kernels themselves).
                                  * Non-NULL: pcl_step_stats runs as ONE launch (plan folded into the scan's last block).
                                  * Words [0,8): counters; word 7 != 0 turns on the diagnostic timeline in words [16,1024)
                                  * (csrc/pcl_common.cuh: per-kernel min start / max end of %globaltimer) */
  /* element types (PCL_DT_*; 0 = fp32, so a zero-initialised descriptor reads fp32).  embed_dtype != 0: `embed` and
   * `grad_embed` point to 2-byte elements; seg_dtype != 0: `seg` does.  The sampled anchors, the loss and every scratch
   * buffer stay fp32. */
  int32_t embed_dtype, seg_dtype;
  /* a10: k >= 1 keeps the k hardest negatives of every anchor (pcl_infonce_topk_fwd / pcl_infonce_tc_topk_fwd on the
   * step's sweep), 0 = all negatives (the reference), < 0 is PCL_ERR_ARG.  Needs an fp32 embed.  topk_scratch: the
   * sweep's pcl_topk_scratch_u32 / pcl_tc_topk_scratch_u32 uint32 words (radix bins + the selection state, which the
   * backward reads: one step owns it from its forward to its backward). */
  int32_t topk_negatives;
  uint32_t* topk_scratch;
} pcl_step_desc;

/* pcl_step_forward: pcl_select_gather + pcl_infonce_fwd (pcl_infonce_tc_fwd with precision 1); with topk_negatives the
 * selection + gather, then the top-k forward of the step's sweep.  pcl_step_backward: the backward sweep (the top-k one
 * with topk_negatives) + pcl_scatter_grad. */
int pcl_step_stats(const pcl_step_desc* d, void* stream);      /* pcl_class_stats + pcl_plan_anchors      */
int pcl_step_forward(const pcl_step_desc* d, void* stream);
int pcl_step_backward(const pcl_step_desc* d, const float* grad_loss, void* stream);
/* Same backward for a grad_embed buffer the caller has already zero-filled (e.g. on a second stream, overlapped with
 * the forward: the 268 MB fill is the HBM floor of the step, the selection and sweep kernels are latency-bound): runs
 * the backward sweep and scatters only the sampled columns.  Nothing else of grad_embed is written.  Not for top-k
 * steps (PCL_ERR_UNSUPPORTED): their backward writes the dense gradient itself. */
int pcl_step_backward_prezeroed(const pcl_step_desc* d, const float* grad_loss, void* stream);
/* pcl_step_backward (csrc/pcl_step.cu:149) with the anchor columns as its output instead of the dense grad_embed, which
 * is not touched: d loss / d embed is zero outside the A <= max_samples sampled pixels.  cols (max_samples, D) fp32:
 * row s < A holds the values pcl_step_backward writes at the anchor's pixel (bit-identical for an fp32 embed; for a
 * half embed, the fp32 values before its rounding), col_pix[s] = b*h*w + pix; rows s >= A are zero with col_pix -1.  A
 * stays on the device (no host sync).  Every mode of pcl_step_backward: exact and tensor sweeps, top-k, normalize,
 * bank. */
int pcl_step_backward_cols(const pcl_step_desc* d, const float* grad_loss, float* cols, int32_t* col_pix, void* stream);

/* CUDA-graph capture of a step (SURVEY §8f row 4).  The three calls above neither allocate nor synchronise, so a
 * stats -> forward -> backward sequence can be captured with cudaStreamBeginCapture / replayed with cudaGraphLaunch.
 * Kernel arguments are frozen in a captured graph, so the by-value sampling seed (pcl_step_desc.seed) would repeat:
 * call pcl_step_ranks between pcl_step_stats and pcl_step_forward and pass its output as pcl_step_desc.ranks.  It
 * draws the anchor ranks with the selection's own device RNG from (d->seed, *step_counter) and increments the
 * counter in device memory, so every replay samples a fresh anchor set (replaces torch.randperm of
 * lib/loss/loss_contrast.py:79-82 exactly like the eager device RNG does).
 *   step_counter  1 uint64 in device memory (caller-initialised, e.g. 0), read and incremented on the stream
 *   ranks         max_samples int32 */
int pcl_step_ranks(const pcl_step_desc* d, uint64_t* step_counter, int32_t* ranks, void* stream);
/* pcl_step_forward for captured sequences without the separate rank draw: the selection kernel draws the anchors from
 * *step_counter itself (same bijection and seed formula as pcl_step_ranks) and the forward's last kernel advances it. */
int pcl_step_forward_ctr(const pcl_step_desc* d, uint64_t* step_counter, void* stream);

/* Fused small-anchor step (self-contrast, no bank, tensor path, D = 256, max_samples <= 1024, no in-kernel normalise:
 * the shape of BASELINE configs[1]).  Four launches for the whole loss step instead of eleven:
 *   pcl_step_stats          label/argmax scan + totals + plan in one launch (d->sync != NULL)
 *   pcl_step_fused_select   selection + gather; anchor ranks drawn from *step_counter (captured sequences), or from
 *                           d->seed / d->ranks when step_counter is NULL
 *   pcl_step_fused_loss     ONE kernel for the InfoNCE forward and backward (logits stay in registers;
 *                           csrc/pcl_infonce_fused.cu)
 *   pcl_step_fused_scatter  sum of the per-column-tile gradient partials + scatter of the A sampled rows into
 *                           d->grad_embed; advances *step_counter.
 * The dense gradient d->grad_embed must be zero outside the A sampled columns.  Two ways:
 *   full fill     pcl_step_fused_fill before the scatter, e.g. on a second stream forked AFTER the selection: the 268 MB fill
 *                 saturates HBM and multiplies the latency of every DRAM read issued next to it (scan, selection), while
 *                 the L2-resident InfoNCE kernel hides behind it;
 *   sparse reset  prev_rows != NULL (1 + 2 * max_samples int32, zero before the first call, owned by the step): the buffer
 *                 persists between steps, zero-filled ONCE by the caller; the selection kernel clears exactly the entries
 *                 the previous step scattered and the scatter records its own.  The caller must not write the buffer.
 * d->sync is required.  pcl_step_fused_supported: 1 if the descriptor qualifies, else 0.  A top-k step
 * (topk_negatives != 0) never qualifies, and every pcl_step_fused_* call returns PCL_ERR_UNSUPPORTED for it. */
int pcl_step_fused_supported(const pcl_step_desc* d);
int pcl_step_fused_select(const pcl_step_desc* d, const uint64_t* step_counter, const int32_t* prev_rows, void* stream);
int pcl_step_fused_loss(const pcl_step_desc* d, void* stream);
int pcl_step_fused_scatter(const pcl_step_desc* d, const float* grad_scale, uint64_t* step_counter, int32_t* prev_rows,
                           void* stream);
/* pcl_step_fused_scatter (csrc/pcl_step.cu:200) with the anchor columns as its output, in the layout of
 * pcl_step_backward_cols: cols (max_samples, 256) fp32, row s < A = the values the scatter writes at the anchor's pixel
 * (the same fixed-order sum of the live per-column-tile partials, times *grad_scale: bit-identical for an fp32 embed, the
 * fp32 values before the rounding for a half embed), col_pix[s] = b*h*w + pix; rows s >= A are zero with col_pix -1, so
 * every row is written on every call.  d->grad_embed is not read or written: no fill is needed.  Advances *step_counter
 * (may be NULL).  sparse reset has no meaning here (no dense buffer). */
int pcl_step_fused_cols(const pcl_step_desc* d, const float* grad_scale, uint64_t* step_counter, float* cols,
                        int32_t* col_pix, void* stream);
int pcl_step_fused_fill(const pcl_step_desc* d, void* stream);   /* zero-fill of d->grad_embed (B*D*h*w elements of
                                                                    d->embed_dtype) */
/* Zero-fill `bytes` (multiple of 16, 16-byte aligned) with 16-byte stores on the engine's own fill kernel. */
int pcl_fill_zero(void* ptr, uint64_t bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PCL_H_ */
