// a10 (SURVEY §8): C entry points of the per-anchor top-k hard-negative selection on the exact fp32 sweep.
//
// Not in the reference code (lib/loss/loss_contrast.py:116-117 sums ALL negatives); default off.  The kernels are modes
// of the shared SIMT sweep (k_sweep<H1..H3, NEGW, BWDW> in pcl_infonce_simt.cu) and the radix-level scan of
// pcl_topk.cuh; the loss step reaches them through pcl_step_desc.topk_negatives.  These are the calls on explicit
// operands, thin wrappers of the sweep's forward / backward with k >= 1.
#include "pcl_common.cuh"
#include "pcl_simt_tile.cuh"
#include "pcl_topk.cuh"

using namespace pcl;

extern "C" int64_t pcl_topk_scratch_u32(const pcl_sweep_desc* d) {
  if (!d) return PCL_ERR_ARG;
  pcl_sweep_sizes_t ss;
  int st = pcl_sweep_sizes(d, &ss);
  if (st != PCL_OK) return st;
  const int64_t a_pad = (int64_t)ss.row_tiles * TM;
  return a_pad * TK_BINS + 4 * (int64_t)d->a_rows;
}

// k < 1 maps to -1: an error here, not "all negatives" (k = 0 of the sweep)
extern "C" int pcl_infonce_topk_fwd(const pcl_sweep_desc* d, int32_t k, uint32_t* scratch, float* partials,
                                    float* rowstats, float* loss, void* stream) {
  return pcl::simt_fwd_ex(d, k < 1 ? -1 : k, scratch, partials, rowstats, loss, stream, nullptr);
}

extern "C" int pcl_infonce_topk_bwd(const pcl_sweep_desc* d, int32_t k, uint32_t* scratch, const float* rowstats,
                                    const float* grad_loss, float* dpartials, float* dA, void* stream) {
  return pcl::simt_bwd_ex(d, k < 1 ? -1 : k, scratch, rowstats, grad_loss, dpartials, dA, stream);
}
