// Fused segmentation losses of the contrast wrappers: the plain CE (first part of this file), the RMI loss of
// contrast.use_rmi (second part), the Lovasz-softmax term of FSCELOVASZLoss (third part) and the OHEM cross-entropy of
// FSOhemCELoss (fourth part, which runs the first part's tile kernels with their OHEM flag set).  All up-sample the
// logits bilinearly inside the kernels and share the tile geometry and transposed bilinear map of pcl_upsample.cuh.
//
// Fused segmentation cross-entropy of ContrastCELoss.forward (SURVEY §8f row 1, the next row after the contrast path):
// replaces  F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True)  +  nn.CrossEntropyLoss(weight, ignore_index,
// reduction='mean')  (lib/loss/loss_contrast.py:180-181, lib/loss/loss_helper.py:169-212) without materialising the
// (B,K,Himg,Wimg) up-sampled logits (318 MB at B=8, K=19, 512x1024) or its log-softmax / gradient copies.
//   k_segce_fwd  one thread per label pixel: 4-neighbour bilinear logits for all K classes (two sweeps: max, then
//                sum of exp), NLL of the target class, log-sum-exp kept per pixel (B*Himg*Wimg floats) for backward;
//                per-CTA partial sums -> k_segce_finalize (fixed order: bit-reproducible)
//   k_segce_bwd  one thread per logit seg[b,c,y,x]: gathers over the label pixels in its bilinear footprint
//                (weight * (softmax - onehot)), no atomics: deterministic — the gather kernel, used for down-sampling
//                geometries; the default up-sampling geometry runs k_segce_bwd_tile, which accumulates the source
//                cells shared by up to 4 neighbouring tiles with fp32 global atomics: its dseg is reproducible only to
//                the last ulp or two (summation order of <= 4 addends), which the parity tolerance (1e-5 max|g|) covers
//   k_segce_fwd_bwd_tile  both in one tile pass, when the upstream gradient is a device scalar that exists before the
//                pass (a captured terminal loss): the forward's lse and partials in the backward tile's pre, the unscaled
//                gradient in its fill, then k_segce_finalize and k_segce_scale (dseg *= grad / sum(w))
// HBM: reads seg (B*K*h*w*4) + labels (B*Himg*Wimg*8), writes lse (B*Himg*Wimg*4); backward re-reads them and writes
// dseg (the one-pass form writes no lse and reads the labels once, then reads and writes dseg once more to scale it).
// Everything else stays in L1/L2 (a 4x4 block of label pixels shares its 4 source logits).
#include "pcl_upsample.cuh"
#include <math_constants.h>

namespace pcl {

struct SegCeArgs : UpGeom {
  const float* seg; const int64_t* target; const float* weight;
  int ignore_index;
};

constexpr int CE_THREADS = 256;

// Fixed-order sums of two per-CTA partial arrays by a 1024-thread CTA: thread i accumulates entries i, i + 1024, ... in
// TA / TB, then a 512 -> 1 tree; thread 0 then runs done(total_a, total_b).  The totals reach done as references to
// shared memory, so they are read where done uses them.  The finalisers built on it are bit-reproducible.
template <class TA, class TB, class PA, class PB, class Done>
__device__ __forceinline__ void block_sum2_1024(const PA* pa, const PB* pb, int64_t n, Done done) {
  __shared__ TA s_a[1024];
  __shared__ TB s_b[1024];
  TA va = 0;
  TB vb = 0;
  for (int64_t i = threadIdx.x; i < n; i += 1024) { va += pa[i]; vb += pb[i]; }
  s_a[threadIdx.x] = va; s_b[threadIdx.x] = vb;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) { s_a[threadIdx.x] += s_a[threadIdx.x + o]; s_b[threadIdx.x] += s_b[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) done(s_a[0], s_b[0]);
}

// Exclusive scan of one int per thread of a 1024-thread CTA, in a fixed order: warp shuffle-up scans, then one warp over
// the 32 warp totals (s_w: 32 ints of shared memory).  Every thread calls it (it contains barriers).
__device__ __forceinline__ int block_exclusive_scan_1024(int v, int* s_w) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = v;                                                      // warp inclusive scan
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const int wv = s_w[lane];
    int wi = wv;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += u;
    }
    s_w[lane] = wi - wv;                                             // exclusive warp offsets
  }
  __syncthreads();
  return s_w[wid] + incl - v;
}

// Backward tile skeleton of the up-sampling losses: one CTA = a 32 x 8 tile of label pixels of one image, classes in
// chunks of kc.  Dynamic shared memory: G [kc][BTY][BT] | Hx [kc][BTY][SRC_MAX] | S [kc][pitch] source patch.
//   pre(g, px, S)             once, after the tile tables (a pass over the classes that the chunks need first)
//   per chunk: the source patch is staged; fill(c0, cn, px, S, G) writes G[cc][ty][tx], the gradient w.r.t. the
//   (virtual) up-sampled logits of the chunk; the transposed bilinear map takes it into dseg (up_tile_flush)
// PRE_STAGES: when one chunk holds every class (K <= kc), pre leaves that chunk staged in S and the loop does not stage
// it again.
template <bool PRE_STAGES = false, class Pre, class Fill>
__device__ __forceinline__ void up_bwd_tile(const UpGeom& a, const float* seg, float* dseg, int kc, int pitch, Pre pre,
                                            Fill fill) {
  extern __shared__ float sm[];
  float* G = sm;                                   // [kc][BTY][BT]
  float* Hx = G + (size_t)kc * BTY * BT;           // [kc][BTY][SRC_MAX]
  float* S = Hx + (size_t)kc * BTY * SRC_MAX;      // [kc][pitch] source patch
  __shared__ int s_y0[BTY], s_y1[BTY], s_x0[BT], s_x1[BT];
  __shared__ float s_ly[BTY], s_lx[BT];
  __shared__ float s_wx[SRC_MAX * (BT + 1)], s_wy[SRC_MAX * (BTY + 1)];
  __shared__ short s_xlo[SRC_MAX], s_xhi[SRC_MAX], s_ylo[SRC_MAX], s_yhi[SRC_MAX];
  const int b = blockIdx.z;
  const int64_t hw = (int64_t)a.h * a.w;
  const UpTile g = up_tile_coords(blockIdx.x * BT, blockIdx.y * BTY, a.H, a.W, a.h, a.w, a.ry, a.rx, s_y0, s_y1, s_ly,
                                  s_x0, s_x1, s_lx);
  const UpPix px = up_pix(g, threadIdx.x & (BT - 1), threadIdx.x >> 5, s_y0, s_y1, s_ly, s_x0, s_x1, s_lx);
  up_tile_tables(g, a.ry, a.rx, s_y0, s_y1, s_ly, s_x0, s_x1, s_lx, s_wx, s_wy, s_xlo, s_xhi, s_ylo, s_yhi);
  pre(g, px, S);
  __syncthreads();
  for (int c0 = 0; c0 < a.K; c0 += kc) {
    const int cn = min(kc, a.K - c0);
    if (!PRE_STAGES || cn < a.K) {
      up_stage(a, seg, b, c0, cn, g.ys_base, g.xs_base, g.ys_n, g.xs_n, pitch, S);
      __syncthreads();
    }
    fill(c0, cn, px, S, G);
    __syncthreads();
    up_tile_flush(g, cn, G, Hx, s_wx, s_wy, s_xlo, s_xhi, s_ylo, s_yhi, dseg + ((int64_t)b * a.K + c0) * hw, hw, a.w);
    __syncthreads();
  }
}

// Per-pixel outputs of the OHEM forward (OHEM = true, fourth part of this file); the plain CE leaves them unused.
struct OhemPix {
  float* p;                     // p_t = softmax of the target class; NaN at a pixel that does not count
  float* wnll;                  // w_t * nll
  int* counts;                  // {counted pixels n, pixels with p_t < thresh}
  float thresh;                 // fp32(thresh)
};

// Forward, tile formulation: the <= (32*ry+2) x (32*rx+2) source logits of the tile are staged in shared memory per class
// chunk; every thread (one label pixel) runs an online log-sum-exp over the classes from shared memory.  With OHEM the
// per-CTA partial sums give way to the per-pixel p_t and w_t * nll, and the two counts go to integer atomics.
template <bool OHEM>
__global__ void __launch_bounds__(BT * BTY)
k_segce_fwd(SegCeArgs a, float* __restrict__ lse_out, float* __restrict__ part_nll, float* __restrict__ part_w, int pitch,
            int kc, OhemPix o) {
  extern __shared__ float sm[];                    // [kc][pitch] source patch
  __shared__ float s_n[BT * BTY / 32], s_w[BT * BTY / 32];
  __shared__ int s_y0[BTY], s_y1[BTY], s_x0[BT], s_x1[BT];
  __shared__ float s_ly[BTY], s_lx[BT];
  const int tx = threadIdx.x & (BT - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int X0 = blockIdx.x * BT, Y0 = blockIdx.y * BTY;
  const int x = X0 + tx, y = Y0 + ty;
  const int64_t HWo = (int64_t)a.H * a.W;
  const UpTile g = up_tile_coords(X0, Y0, a.H, a.W, a.h, a.w, a.ry, a.rx, s_y0, s_y1, s_ly, s_x0, s_x1, s_lx);
  const UpPix px = up_pix(g, tx, ty, s_y0, s_y1, s_ly, s_x0, s_x1, s_lx);
  const bool inside = x < a.W && y < a.H;
  int64_t t = -1;
  if (inside) t = a.target[(int64_t)b * HWo + (int64_t)y * a.W + x];
  float m = -CUDART_INF_F, se = 0.f, vt = 0.f;
  for (int c0 = 0; c0 < a.K; c0 += kc) {
    const int cn = min(kc, a.K - c0);
    up_stage(a, a.seg, b, c0, cn, g.ys_base, g.xs_base, g.ys_n, g.xs_n, pitch, sm);
    __syncthreads();
    for (int cc = 0; cc < cn; ++cc) {
      const float v = up_logit(px, sm + cc * pitch);
      if (v > m) { se = se * __expf(m - v) + 1.f; m = v; }     // online log-sum-exp
      else       { se += __expf(v - m); }
      if (c0 + cc == (int)t) vt = v;
    }
    __syncthreads();
  }
  float nll = 0.f, wt = 0.f;
  if (inside) {
    const float lse = m + __logf(se);
    lse_out[(int64_t)b * HWo + (int64_t)y * a.W + x] = lse;
    if (t != (int64_t)a.ignore_index && t >= 0 && t < a.K) {
      const float wc = a.weight ? a.weight[t] : 1.f;
      nll = wc * (lse - vt);
      wt = wc;
    }
    if constexpr (OHEM) {
      const int64_t q = (int64_t)b * HWo + (int64_t)y * a.W + x;
      const bool counted = t != (int64_t)a.ignore_index && t >= 0 && t < a.K;
      const float p = counted ? __expf(vt - m) / se : CUDART_NAN_F;
      o.p[q] = p;
      o.wnll[q] = nll;
      nll = counted ? 1.f : 0.f;                   // the two counts take the partial sums' place (exact in fp32)
      wt = p < o.thresh ? 1.f : 0.f;
    }
  }
  nll = warp_sum(nll); wt = warp_sum(wt);
  if ((threadIdx.x & 31) == 0) { s_n[threadIdx.x >> 5] = nll; s_w[threadIdx.x >> 5] = wt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float an = 0.f, aw = 0.f;
    for (int i = 0; i < BT * BTY / 32; ++i) { an += s_n[i]; aw += s_w[i]; }      // fixed order
    if constexpr (OHEM) {
      if (an > 0.f) { atomicAdd(&o.counts[0], (int)an); atomicAdd(&o.counts[1], (int)aw); }
    } else {
      const int64_t blk = ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
      part_nll[blk] = an;
      part_w[blk] = aw;
    }
  }
}

__global__ void __launch_bounds__(1024)
k_segce_finalize(const float* __restrict__ part_nll, const float* __restrict__ part_w, int64_t n, float* __restrict__ out) {
  block_sum2_1024<double, double>(part_nll, part_w, n, [&](const double& an, const double& aw) {
    out[0] = (float)(an / aw);                  // 'mean' reduction: sum(w_t * nll) / sum(w_t) over non-ignored pixels
    out[1] = (float)aw;
  });
}

// Backward, tile formulation (up_bwd_tile): per chunk, a thread per label pixel computes
// G[c] = coef * w_t * (softmax_c - [c == t]) from the staged source patch; then the transposed bilinear map into dseg.
// Each (pixel, class) softmax is evaluated once (the per-logit gather below needs 16x as many); the map only visits the
// label columns / rows inside the footprint of their source cell.
// With OHEM, fin is the OHEM state (fin[1] the denominator, fin[2] the threshold) and only the pixels whose stored
// p_t (ohem_p) lies below the threshold carry a gradient: the forward's selection, read back rather than recomputed.
template <bool OHEM>
__global__ void __launch_bounds__(BT * BTY, 5)     // 5 CTAs per SM: holds the kernel at 48 registers
k_segce_bwd_tile(SegCeArgs a, const float* __restrict__ lse, const float* __restrict__ fin,
                 const float* __restrict__ grad_out, const float* __restrict__ ohem_p, float* __restrict__ dseg, int kc,
                 int pitch) {
  const int tx = threadIdx.x & (BT - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int x = blockIdx.x * BT + tx, y = blockIdx.y * BTY + ty;
  const int64_t HWo = (int64_t)a.H * a.W;
  const float scale = (grad_out ? grad_out[0] : 1.f) / fin[1];
  int64_t t = -1;
  float lse_p = 0.f, coef = 0.f;
  if (x < a.W && y < a.H) {
    t = a.target[(int64_t)b * HWo + (int64_t)y * a.W + x];
    if (t != (int64_t)a.ignore_index && t >= 0 && t < a.K &&
        (!OHEM || ohem_p[(int64_t)b * HWo + (int64_t)y * a.W + x] < fin[2])) {
      coef = scale * (a.weight ? a.weight[t] : 1.f);
      lse_p = lse[(int64_t)b * HWo + (int64_t)y * a.W + x];
    } else {
      t = -1;
    }
  }
  up_bwd_tile(a, a.seg, dseg, kc, pitch, [](const UpTile&, const UpPix&, float*) {},
              [&](int c0, int cn, const UpPix& px, const float* S, float* G) {
    for (int cc = 0; cc < cn; ++cc) {
      float gv = 0.f;
      if (t >= 0) {
        const float v = up_logit(px, S + cc * pitch);
        gv = coef * (__expf(v - lse_p) - ((c0 + cc) == (int)t ? 1.f : 0.f));
      }
      G[((size_t)cc * BTY + ty) * BT + tx] = gv;
    }
  });
}

// Forward and backward in one tile pass (up_bwd_tile), for a caller whose upstream gradient is a device scalar that
// exists when the pass runs (a captured terminal loss).  pre runs k_segce_fwd's online log-sum-exp over every class
// (same class order, same up_logit, same __expf / __logf), so the lse, nll and w_t of every pixel and the per-CTA
// partials, written in k_segce_fwd's order and layout, are its bits; fill writes the unscaled w_t * (softmax_c - [c == t]).
// k_segce_finalize sums the partials and k_segce_scale applies grad / sum(w).  No per-pixel lse goes to HBM and the
// labels are read once; at K <= kc the patch pre stages serves the fill too.
__global__ void __launch_bounds__(BT * BTY, 4)     // 4 CTAs per SM: 64 registers
k_segce_fwd_bwd_tile(SegCeArgs a, float* __restrict__ part_nll, float* __restrict__ part_w, float* __restrict__ dseg,
                     int kc, int pitch) {
  __shared__ float s_n[BT * BTY / 32], s_w[BT * BTY / 32];
  const int tx = threadIdx.x & (BT - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int x = blockIdx.x * BT + tx, y = blockIdx.y * BTY + ty;
  const int64_t HWo = (int64_t)a.H * a.W;
  const bool inside = x < a.W && y < a.H;
  int64_t t = -1;
  if (inside) t = a.target[(int64_t)b * HWo + (int64_t)y * a.W + x];
  float lse = 0.f, wt = 0.f;
  up_bwd_tile<true>(a, a.seg, dseg, kc, pitch, [&](const UpTile& g, const UpPix& px, float* S) {
    float m = -CUDART_INF_F, se = 0.f, vt = 0.f;
    for (int c0 = 0; c0 < a.K; c0 += kc) {
      const int cn = min(kc, a.K - c0);
      if (c0 > 0) __syncthreads();                 // the previous chunk is read
      up_stage(a, a.seg, b, c0, cn, g.ys_base, g.xs_base, g.ys_n, g.xs_n, pitch, S);
      __syncthreads();
      for (int cc = 0; cc < cn; ++cc) {
        const float v = up_logit(px, S + cc * pitch);
        if (v > m) { se = se * __expf(m - v) + 1.f; m = v; }     // online log-sum-exp
        else       { se += __expf(v - m); }
        if (c0 + cc == (int)t) vt = v;
      }
    }
    float nll = 0.f;
    bool counted = false;
    if (inside) {
      lse = m + __logf(se);
      if (t != (int64_t)a.ignore_index && t >= 0 && t < a.K) {
        const float wc = a.weight ? a.weight[t] : 1.f;
        nll = wc * (lse - vt);
        wt = wc;
        counted = true;
      }
    }
    if (!counted) t = -1;                          // no gradient
    float an = warp_sum(nll), aw = warp_sum(wt);
    if ((threadIdx.x & 31) == 0) { s_n[threadIdx.x >> 5] = an; s_w[threadIdx.x >> 5] = aw; }
    __syncthreads();
    if (threadIdx.x == 0) {
      an = 0.f; aw = 0.f;
      for (int i = 0; i < BT * BTY / 32; ++i) { an += s_n[i]; aw += s_w[i]; }      // fixed order
      const int64_t blk = ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
      part_nll[blk] = an;
      part_w[blk] = aw;
    }
  }, [&](int c0, int cn, const UpPix& px, const float* S, float* G) {
    for (int cc = 0; cc < cn; ++cc) {
      float gv = 0.f;
      if (t >= 0) {
        const float v = up_logit(px, S + cc * pitch);
        gv = wt * (__expf(v - lse) - ((c0 + cc) == (int)t ? 1.f : 0.f));
      }
      G[((size_t)cc * BTY + ty) * BT + tx] = gv;
    }
  });
}

// dseg *= grad / sum(w) after k_segce_fwd_bwd_tile.  Every pixel ignored (sum(w) == 0, the loss is NaN): dseg stays the
// zeros the tile pass left, as the two-kernel backward leaves it (no 0 * inf).
__global__ void __launch_bounds__(CE_THREADS)
k_segce_scale(float* __restrict__ dseg, int64_t n, const float* __restrict__ fin, const float* __restrict__ grad_out) {
  const float aw = fin[1];
  if (aw == 0.f) return;
  const float scale = (grad_out ? grad_out[0] : 1.f) / aw;
  const int64_t stride = (int64_t)gridDim.x * CE_THREADS;
  const int64_t n4 = (reinterpret_cast<uintptr_t>(dseg) & 15) ? 0 : n >> 2;    // float4 when 16-byte aligned
  float4* d4 = reinterpret_cast<float4*>(dseg);
  for (int64_t i = (int64_t)blockIdx.x * CE_THREADS + threadIdx.x; i < n4; i += stride) {
    float4 v = d4[i];
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    d4[i] = v;
  }
  for (int64_t i = 4 * n4 + (int64_t)blockIdx.x * CE_THREADS + threadIdx.x; i < n; i += stride) dseg[i] *= scale;
}

// General backward (any scale, e.g. label grid smaller than the logits): one thread per logit gathers over the label
// pixels in its bilinear footprint.  Deterministic, but evaluates every (pixel, class) softmax up to 16 times; the tile
// kernel above is used whenever the label grid is at least as large as the logit grid (the reference's case).
__device__ __forceinline__ void footprint(int s, float r, int out_size, int& lo, int& hi) {
  if (r <= 0.f) { lo = 0; hi = out_size - 1; return; }
  lo = (int)floorf(((float)s - 1.f) / r) - 1;
  hi = (int)ceilf(((float)s + 1.f) / r) + 1;
  if (lo < 0) lo = 0;
  if (hi > out_size - 1) hi = out_size - 1;
}

__global__ void __launch_bounds__(CE_THREADS)
k_segce_bwd_gather(SegCeArgs a, const float* __restrict__ lse, const float* __restrict__ fin,
                   const float* __restrict__ grad_out, float* __restrict__ dseg) {
  const int64_t hw = (int64_t)a.h * a.w;
  const int64_t e = (int64_t)blockIdx.x * CE_THREADS + threadIdx.x;
  const int bc = blockIdx.y;
  if (e >= hw) return;
  const int b = bc / a.K, c = bc - b * a.K;
  const int ys = (int)(e / a.w), xs = (int)(e - (int64_t)ys * a.w);
  const int64_t HWo = (int64_t)a.H * a.W;
  const float scale = (grad_out ? grad_out[0] : 1.f) / fin[1];
  const float* p = a.seg + ((int64_t)b * a.K + c) * hw;
  int ylo, yhi, xlo, xhi;
  footprint(ys, a.ry, a.H, ylo, yhi);
  footprint(xs, a.rx, a.W, xlo, xhi);
  float acc = 0.f;
  for (int y = ylo; y <= yhi; ++y) {
    int y0, y1; float ly;
    src_coord(y, a.ry, a.h, y0, y1, ly);
    float wy = 0.f;
    if (y0 == ys) wy += 1.f - ly;
    if (y1 == ys) wy += ly;
    if (wy == 0.f) continue;
    for (int x = xlo; x <= xhi; ++x) {
      int x0, x1; float lx;
      src_coord(x, a.rx, a.w, x0, x1, lx);
      float wx = 0.f;
      if (x0 == xs) wx += 1.f - lx;
      if (x1 == xs) wx += lx;
      if (wx == 0.f) continue;
      const int64_t pix = (int64_t)y * a.W + x;
      const int64_t t = a.target[(int64_t)b * HWo + pix];
      if (t == (int64_t)a.ignore_index || t < 0 || t >= a.K) continue;
      const float v = (1.f - ly) * (1.f - lx) * p[(int64_t)y0 * a.w + x0] + (1.f - ly) * lx * p[(int64_t)y0 * a.w + x1] +
                      ly * (1.f - lx) * p[(int64_t)y1 * a.w + x0] + ly * lx * p[(int64_t)y1 * a.w + x1];
      const float prob = expf(v - lse[(int64_t)b * HWo + pix]);
      const float wc = a.weight ? a.weight[t] : 1.f;
      acc += wy * wx * wc * (prob - (c == (int)t ? 1.f : 0.f));
    }
  }
  // every pixel ignored (weight sum 0): acc is 0 and scale infinite; the gradient is 0, as the tile kernels leave it
  dseg[((int64_t)b * a.K + c) * hw + e] = fin[1] == 0.f ? 0.f : acc * scale;
}

}  // namespace pcl

using namespace pcl;

static int make_ce(const float* seg, const int64_t* target, const float* weight, int B, int K, int h, int w, int H, int W,
                   int ignore_index, SegCeArgs* a) {
  if (!seg || !target) return PCL_ERR_ARG;
  const int st = up_geometry(B, K, h, w, H, W, a);
  if (st != PCL_OK) return st;
  a->seg = seg; a->target = target; a->weight = weight; a->ignore_index = ignore_index;
  return PCL_OK;
}

template <bool OHEM>
static int segce_fwd_launch(const SegCeArgs& a, float* lse, float* pn, float* pw, OhemPix o, cudaStream_t s) {
  UpPlan pl;
  const int st = up_fwd_plan(a, up_patch_pitch(a, BTY, BT), 0, &pl);
  if (st != PCL_OK) return st;
  PCL_SMEM_OPT_IN(k_segce_fwd<OHEM>, 200 * 1024);
  k_segce_fwd<OHEM><<<dim3((unsigned)ceil_div(a.W, BT), (unsigned)ceil_div(a.H, BTY), a.B), BT * BTY, pl.smem, s>>>(
      a, lse, pn, pw, pl.pitch, pl.kc, o);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

// Launch plan of the backward tile kernels (up_bwd_tile): dseg is zeroed here (the kernel accumulates into it); kc
// classes per pass, at most KC_BWD_MAX, fewer while G + Hx + the source patch (kc * (BTY*BT + BTY*SRC_MAX + pitch)
// floats) exceed 200 KB.  The kernel is a template argument because PCL_SMEM_OPT_IN keeps one flag per instantiation:
// every kernel opts in on its own, k_segce_bwd_tile<false> and <true> included (they have the same type).
template <auto Kernel, class Args, class... P>
static int up_bwd_launch(const Args& a, cudaStream_t s, float* dseg, P... p) {
  PCL_CUDA(cudaMemsetAsync(dseg, 0, (size_t)a.B * a.K * a.h * a.w * sizeof(float), s));
  const int pitch = up_patch_pitch(a, BTY, BT);
  int kc = a.K < KC_BWD_MAX ? a.K : KC_BWD_MAX;
  while (kc > 1 && (size_t)kc * (BTY * BT + BTY * SRC_MAX + pitch) * sizeof(float) > 200 * 1024) --kc;
  const size_t smem = (size_t)kc * (BTY * BT + BTY * SRC_MAX + pitch) * sizeof(float);
  if (smem > 200 * 1024) return PCL_ERR_UNSUPPORTED;
  PCL_SMEM_OPT_IN(Kernel, 200 * 1024);
  Kernel<<<dim3((unsigned)ceil_div(a.W, BT), (unsigned)ceil_div(a.H, BTY), a.B), BT * BTY, smem, s>>>(a, p..., dseg, kc,
                                                                                                      pitch);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int64_t pcl_seg_ce_scratch_floats(int32_t B, int32_t H, int32_t W) {
  const int64_t blocks = (int64_t)ceil_div(H, BTY) * ceil_div(W, BT) * B;
  return (int64_t)B * H * W + 2 * blocks + 2;            // lse | partial nll | partial weight | (loss, weight sum)
}

extern "C" int pcl_seg_ce_fwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K,
                              int32_t h, int32_t w, int32_t H, int32_t W, int32_t ignore_index, float* scratch, float* loss,
                              void* stream) {
  SegCeArgs a;
  int st = make_ce(seg, target, class_weight, B, K, h, w, H, W, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && loss);
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t HWo = (int64_t)H * W;
  const int64_t blocks = (int64_t)ceil_div(H, BTY) * ceil_div(W, BT) * B;
  float* lse = scratch;
  float* pn = scratch + (int64_t)B * HWo;
  float* pw = pn + blocks;
  float* fin = pw + blocks;
  st = segce_fwd_launch<false>(a, lse, pn, pw, OhemPix{}, s);
  if (st != PCL_OK) return st;
  k_segce_finalize<<<1, 1024, 0, s>>>(pn, pw, blocks, fin);
  PCL_LAUNCH_CHECK();
  PCL_CUDA(cudaMemcpyAsync(loss, fin, sizeof(float), cudaMemcpyDeviceToDevice, s));
  return PCL_OK;
}

extern "C" int pcl_seg_ce_bwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K,
                              int32_t h, int32_t w, int32_t H, int32_t W, int32_t ignore_index, const float* scratch,
                              const float* grad_loss, float* dseg, void* stream) {
  SegCeArgs a;
  int st = make_ce(seg, target, class_weight, B, K, h, w, H, W, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && dseg);
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t HWo = (int64_t)H * W;
  const int64_t blocks = (int64_t)ceil_div(H, BTY) * ceil_div(W, BT) * B;
  const float* lse = scratch;
  const float* fin = scratch + (int64_t)B * HWo + 2 * blocks;
  const int64_t hw = (int64_t)h * w;
  if (H < h || W < w) {                                     // down-sampling: general gather kernel
    k_segce_bwd_gather<<<dim3((unsigned)ceil_div64(hw, CE_THREADS), B * K), CE_THREADS, 0, s>>>(a, lse, fin, grad_loss, dseg);
    PCL_LAUNCH_CHECK();
    return PCL_OK;
  }
  return up_bwd_launch<k_segce_bwd_tile<false>>(a, s, dseg, lse, fin, grad_loss, (const float*)nullptr);
}

// One tile pass where one class chunk holds every class (K <= KC_BWD_MAX): the pass then stages the patch once instead of
// twice and the labels and the lse stay out of HBM.  With several chunks both passes stage every chunk anyway, and the
// scale pass over dseg made the one-pass form slower than the two kernels (DESIGN §4, ADE20K shape): pcl_seg_ce_fwd's
// and pcl_seg_ce_bwd's kernels run there, with the lse in front of the partials in the scratch.
static bool segce_one_pass(int K) { return K <= KC_BWD_MAX; }

extern "C" int64_t pcl_seg_ce_fwd_bwd_scratch_floats(int32_t B, int32_t K, int32_t H, int32_t W) {
  const int64_t blocks = (int64_t)ceil_div(H, BTY) * ceil_div(W, BT) * B;
  return (segce_one_pass(K) ? 0 : (int64_t)B * H * W) + 2 * blocks + 2;     // [lse] | partial nll | partial w | fin
}

extern "C" int pcl_seg_ce_fwd_bwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B,
                                  int32_t K, int32_t h, int32_t w, int32_t H, int32_t W, int32_t ignore_index,
                                  float* scratch, const float* grad_scale, float* loss, float* dseg, void* stream) {
  SegCeArgs a;
  int st = make_ce(seg, target, class_weight, B, K, h, w, H, W, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && loss && dseg);
  if (H < h || W < w) return PCL_ERR_UNSUPPORTED;          // down-sampling: pcl_seg_ce_fwd + pcl_seg_ce_bwd
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t blocks = (int64_t)ceil_div(H, BTY) * ceil_div(W, BT) * B;
  const bool one = segce_one_pass(K);
  float* lse = scratch;
  float* pn = scratch + (one ? 0 : (int64_t)B * H * W);
  float* pw = pn + blocks;
  float* fin = pw + blocks;
  if (!one) {
    st = segce_fwd_launch<false>(a, lse, pn, pw, OhemPix{}, s);
    if (st != PCL_OK) return st;
    k_segce_finalize<<<1, 1024, 0, s>>>(pn, pw, blocks, fin);
    PCL_LAUNCH_CHECK();
    PCL_CUDA(cudaMemcpyAsync(loss, fin, sizeof(float), cudaMemcpyDeviceToDevice, s));
    return up_bwd_launch<k_segce_bwd_tile<false>>(a, s, dseg, (const float*)lse, (const float*)fin, grad_scale,
                                                  (const float*)nullptr);
  }
  st = up_bwd_launch<k_segce_fwd_bwd_tile>(a, s, dseg, pn, pw);
  if (st != PCL_OK) return st;
  k_segce_finalize<<<1, 1024, 0, s>>>(pn, pw, blocks, fin);
  PCL_LAUNCH_CHECK();
  const int64_t n = (int64_t)B * K * h * w;
  const int64_t want = ceil_div64(ceil_div64(n, 4), CE_THREADS);
  const int cap = 8 * num_sms();
  k_segce_scale<<<(unsigned)(want < cap ? (want > 0 ? want : 1) : cap), CE_THREADS, 0, s>>>(dseg, n, fin, grad_scale);
  PCL_LAUNCH_CHECK();
  PCL_CUDA(cudaMemcpyAsync(loss, fin, sizeof(float), cudaMemcpyDeviceToDevice, s));
  return PCL_OK;
}

// ==================================================================================================================
// Fused RMI (Region Mutual Information) segmentation loss, sigmoid path: replaces
//   F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True)  +  RMILoss.forward -> forward_sigmoid ->
//   rmi_lower_bound  (lib/loss/rmi_loss.py:200-402, used by FSRMILoss / FSAuxRMILoss, lib/loss/loss_helper.py:316-369)
// and its autograd backward, without materialising the (B,K,Himg,Wimg) up-sampled logits, one-hot labels and sigmoid
// probabilities, or the float64 (B,K,r*r,n) neighbour vectors (629 MB each at B=8, K=19, 512x1024, r=3, stride 3).
//   k_rmi_pool      one thread per pooled pixel: bilinear logits of its s x s window (source patch staged per class
//                   chunk), sigmoid, max / avg pooling of the probabilities and the label presence, argmax slot; the
//                   BCE of every label pixel (pixels below / right of the last window included); per-CTA partials
//   k_rmi_moments   per (b, c, band of 16 point rows): float64 sums of x, y, x x^T, y y^T, x y^T over the band's
//                   r x r neighbour vectors (fixed order, no atomics: the forward is bit-reproducible)
//   k_rmi_solve     per (b, c): band sums -> centred moments, Cholesky of P and M in float64, log-det; the backward
//                   coefficients 2 dP = A^T M^-1 A and dQ^T = -A^T M^-1 (A = Q P^-1) scaled by the loss weights
//   k_rmi_finalize  BCE and per-class sums -> the scalar loss (fixed order)
//   k_rmi_dpool     dL / d(pooled p) from the r*r neighbour vectors that contain each pooled pixel
//   k_rmi_bwd_tile  per label tile: un-pool (argmax slot or 1/s^2) x sigmoid' + the BCE gradient, then the transposed
//                   bilinear map into dseg (up_tile_flush, shared with the seg CE; fp32 atomics on the <= 4 tiles that
//                   share a source cell, so dseg is reproducible to the last ulp or two, the loss bit for bit)

namespace pcl {

constexpr int RMI_R_MAX = 4;
constexpr int RMI_S_MAX = 4;
constexpr int PT_X = 32, PT_Y = 8;                       // pooled pixels per k_rmi_pool CTA
constexpr int REG_ROWS = PT_Y * RMI_S_MAX + 2 * RMI_S_MAX, REG_COLS = PT_X * RMI_S_MAX + 2 * RMI_S_MAX;
constexpr int MB_Y = 16, MB_X = 64;                      // points per k_rmi_moments band row / column tile
constexpr int MB_PITCH = MB_X + RMI_R_MAX - 1;
constexpr double RMI_ALPHA = 1e-3;                       // _POS_ALPHA
constexpr float RMI_CLIP_MIN = 1e-6f;                    // _CLIP_MIN

static_assert(PT_X * PT_Y == BT * BTY, "k_rmi_pool stages its patch with up_stage (256 threads)");

struct RmiArgs : UpGeom {
  const float* seg; const int64_t* target;
  int r, way, s, pad;           // radius, pool way (0 max, 1 avg), pool size == stride, padding s/2
  int Hp, Wp, nY, nX;           // pooled map, neighbour-vector points (Hp-r+1) x (Wp-r+1)
  float lw, wb, wr;             // loss_weight, BCE weight, RMI weight (lambda_way: lambda, 1-lambda; else 1, lambda)
};

__host__ __device__ constexpr int rmi_entries(int R) { return 2 * R * R + R * R * R * R + R * R * (R * R + 1); }

// label value of a pooled pixel: presence flag (max pool) or count / s^2 in fp32 (avg pool, as F.avg_pool2d)
__device__ __forceinline__ float rmi_label_value(uint8_t cnt, int way, int s) {
  return way == 0 ? (cnt ? 1.f : 0.f) : (float)cnt / (float)(s * s);
}

// ---- forward: pooling + BCE -----------------------------------------------------------------------
__global__ void __launch_bounds__(PT_X * PT_Y)
k_rmi_pool(RmiArgs a, float* __restrict__ P, uint8_t* __restrict__ L, uint8_t* __restrict__ A, float* __restrict__ part_bce,
           int* __restrict__ part_cnt, int pitch, int kc) {
  extern __shared__ float sm[];
  short* lab = reinterpret_cast<short*>(sm);                        // [REG_ROWS][REG_COLS] class id or -1
  float* S = sm + REG_ROWS * REG_COLS / 2;                          // [kc][pitch] source patch
  __shared__ int s_y0[REG_ROWS], s_y1[REG_ROWS], s_x0[REG_COLS], s_x1[REG_COLS];
  __shared__ float s_ly[REG_ROWS], s_lx[REG_COLS];
  __shared__ float s_b[PT_X * PT_Y / 32];
  __shared__ int s_c[PT_X * PT_Y / 32];
  const int tx = threadIdx.x & (PT_X - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int ox0 = blockIdx.x * PT_X, oy0 = blockIdx.y * PT_Y;
  const int ox = ox0 + tx, oy = oy0 + ty;
  const int s = a.s, pad = a.pad;
  // label rows [lo(o), hi(o)) of pooled row o: its window, and for the last one every row below it (BCE only)
  const int oyl = min(oy0 + PT_Y, a.Hp) - 1, oxl = min(ox0 + PT_X, a.Wp) - 1;
  const int R0 = max(0, oy0 * s - pad), C0 = max(0, ox0 * s - pad);
  const int R1 = oyl == a.Hp - 1 ? a.H : min(a.H, (oyl + 1) * s - pad);
  const int C1 = oxl == a.Wp - 1 ? a.W : min(a.W, (oxl + 1) * s - pad);
  const int nr = R1 - R0, nc = C1 - C0;
  for (int i = threadIdx.x; i < nr; i += PT_X * PT_Y) {
    int i0, i1; float l;
    src_coord(R0 + i, a.ry, a.h, i0, i1, l);
    s_y0[i] = i0; s_y1[i] = i1; s_ly[i] = l;
  }
  for (int i = threadIdx.x; i < nc; i += PT_X * PT_Y) {
    int i0, i1; float l;
    src_coord(C0 + i, a.rx, a.w, i0, i1, l);
    s_x0[i] = i0; s_x1[i] = i1; s_lx[i] = l;
  }
  const int64_t HWo = (int64_t)a.H * a.W;
  for (int i = threadIdx.x; i < nr * nc; i += PT_X * PT_Y) {
    const int lr = i / nc, lc = i - lr * nc;
    int64_t t = a.target[(int64_t)b * HWo + (int64_t)(R0 + lr) * a.W + C0 + lc];
    if (t < 0) t = 255;                                              // label[label < 0] = 255
    lab[lr * REG_COLS + lc] = (short)(t < a.K ? t : -1);             // valid: label < num_classes
  }
  __syncthreads();
  const int ys_base = s_y0[0], xs_base = s_x0[0];
  const int ys_n = s_y1[nr - 1] - ys_base + 1, xs_n = s_x1[nc - 1] - xs_base + 1;
  const bool active = oy < a.Hp && ox < a.Wp;
  const int wy0 = oy * s - pad, wx0 = ox * s - pad;                  // window origin (may lie in the padding)
  int ylo = 0, yhi = 0, xlo = 0, xhi = 0;
  if (active) {
    ylo = max(0, wy0) - R0; yhi = (oy == a.Hp - 1 ? a.H : min(a.H, wy0 + s)) - R0;
    xlo = max(0, wx0) - C0; xhi = (ox == a.Wp - 1 ? a.W : min(a.W, wx0 + s)) - C0;
  }
  const int wy1 = wy0 + s - R0, wx1 = wx0 + s - C0;                  // window end, region coordinates
  int nvalid = 0;
  for (int lr = ylo; lr < yhi; ++lr)
    for (int lc = xlo; lc < xhi; ++lc) nvalid += lab[lr * REG_COLS + lc] >= 0;
  float bce = 0.f;
  const int64_t HWp = (int64_t)a.Hp * a.Wp;
  for (int c0 = 0; c0 < a.K; c0 += kc) {
    const int cn = min(kc, a.K - c0);
    up_stage(a, a.seg, b, c0, cn, ys_base, xs_base, ys_n, xs_n, pitch, S);
    __syncthreads();
    if (active) {
      for (int cc = 0; cc < cn; ++cc) {
        const int c = c0 + cc;
        const float* p = S + cc * pitch;
        float pmax = -CUDART_INF_F, psum = 0.f;
        int slot = 0, cnt = 0;
        for (int lr = ylo; lr < yhi; ++lr) {
          const int y0 = s_y0[lr] - ys_base, y1 = s_y1[lr] - ys_base;
          const float ly = s_ly[lr];
          for (int lc = xlo; lc < xhi; ++lc) {
            const int x0 = s_x0[lc] - xs_base, x1 = s_x1[lc] - xs_base;
            const float lx = s_lx[lc];
            const float z = (1.f - ly) * ((1.f - lx) * p[y0 * xs_n + x0] + lx * p[y0 * xs_n + x1]) +
                            ly * ((1.f - lx) * p[y1 * xs_n + x0] + lx * p[y1 * xs_n + x1]);
            const int tv = lab[lr * REG_COLS + lc];
            const float yv = tv == c ? 1.f : 0.f;
            if (tv >= 0) bce += (1.f - yv) * z + fmaxf(-z, 0.f) + log1pf(expf(-fabsf(z)));
            if (lr < wy1 && lc < wx1) {
              const float pr = (tv >= 0 ? 1.f / (1.f + expf(-z)) : 0.f) + RMI_CLIP_MIN;
              if (pr > pmax) { pmax = pr; slot = (lr + R0 - wy0) * s + (lc + C0 - wx0); }   // first maximum wins
              psum += pr;
              cnt += tv == c;
            }
          }
        }
        const int64_t o = ((int64_t)b * a.K + c) * HWp + (int64_t)oy * a.Wp + ox;
        P[o] = a.way == 0 ? pmax : psum / (float)(s * s);
        L[o] = (uint8_t)cnt;
        A[o] = (uint8_t)slot;
      }
    }
    __syncthreads();
  }
  bce = warp_sum(bce);
  nvalid = warp_sum_i(nvalid);
  if ((threadIdx.x & 31) == 0) { s_b[threadIdx.x >> 5] = bce; s_c[threadIdx.x >> 5] = nvalid; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ab = 0.f; int ac = 0;
    for (int i = 0; i < PT_X * PT_Y / 32; ++i) { ab += s_b[i]; ac += s_c[i]; }      // fixed order
    const int64_t blk = ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    part_bce[blk] = ab;
    part_cnt[blk] = ac;
  }
}

// ---- forward: moments ------------------------------------------------------------------------------
// Entry e of the per-(b,c) sum vector: [0, D) sum x_k, [D, 2D) sum y_k, then D*D sum x_k y_l, then the upper triangles
// (k <= l, row-major) of sum x_k x_l and of sum y_k y_l.  Each operand is (plane, offset k) with plane 0 = x, 1 = y, 2 = 1.
template <int R>
__device__ __forceinline__ void rmi_entry(int e, int& pa, int& ka, int& pb, int& kb) {
  constexpr int D = R * R;
  if (e < D) { pa = 0; ka = e; pb = 2; kb = 0; return; }
  if (e < 2 * D) { pa = 1; ka = e - D; pb = 2; kb = 0; return; }
  e -= 2 * D;
  if (e < D * D) { pa = 0; ka = e / D; pb = 1; kb = e % D; return; }
  e -= D * D;
  const int plane = e < D * (D + 1) / 2 ? 0 : 1;
  if (plane) e -= D * (D + 1) / 2;
  int k = 0;
  while (e >= D - k) { e -= D - k; ++k; }
  pa = pb = plane; ka = k; kb = k + e;
}

template <int R>
__global__ void __launch_bounds__(256)
k_rmi_moments(RmiArgs a, const float* __restrict__ P, const uint8_t* __restrict__ L, double* __restrict__ part) {
  constexpr int NE = rmi_entries(R), EPT = (NE + 255) / 256;
  constexpr int ROWS = MB_Y + R - 1;
  __shared__ double pl[3 * (MB_Y + RMI_R_MAX - 1) * MB_PITCH];       // x | y | ones
  const int band = blockIdx.x, bc = blockIdx.y;
  const int py0 = band * MB_Y, npy = min(MB_Y, a.nY - py0);
  const int64_t HWp = (int64_t)a.Hp * a.Wp;
  const float* Pb = P + (int64_t)bc * HWp;
  const uint8_t* Lb = L + (int64_t)bc * HWp;
  constexpr int PLANE = (MB_Y + RMI_R_MAX - 1) * MB_PITCH;
  const double* pa_ptr[EPT];
  const double* pb_ptr[EPT];
  double acc[EPT];
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    acc[i] = 0.0;
    const int e = threadIdx.x + i * 256;
    int pa = 2, ka = 0, pb = 2, kb = 0;
    if (e < NE) rmi_entry<R>(e, pa, ka, pb, kb);
    pa_ptr[i] = pl + pa * PLANE + (ka / R) * MB_PITCH + ka % R;
    pb_ptr[i] = pl + pb * PLANE + (kb / R) * MB_PITCH + kb % R;
  }
  for (int i = threadIdx.x; i < PLANE; i += 256) pl[2 * PLANE + i] = 1.0;
  for (int px0 = 0; px0 < a.nX; px0 += MB_X) {
    const int npx = min(MB_X, a.nX - px0), cols = npx + R - 1;
    __syncthreads();
    for (int i = threadIdx.x; i < ROWS * cols; i += 256) {
      const int rr = i / cols, cc = i - rr * cols;
      double xv = 0.0, yv = 0.0;
      if (rr < npy + R - 1) {
        const int64_t o = (int64_t)(py0 + rr) * a.Wp + px0 + cc;
        xv = (double)rmi_label_value(Lb[o], a.way, a.s);
        yv = (double)Pb[o];
      }
      pl[rr * MB_PITCH + cc] = xv;
      pl[PLANE + rr * MB_PITCH + cc] = yv;
    }
    __syncthreads();
    for (int py = 0; py < npy; ++py)
      for (int px = 0; px < npx; ++px) {
        const int o = py * MB_PITCH + px;
#pragma unroll
        for (int i = 0; i < EPT; ++i) acc[i] = fma(pa_ptr[i][o], pb_ptr[i][o], acc[i]);
      }
  }
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int e = threadIdx.x + i * 256;
    if (e < NE) part[((int64_t)bc * gridDim.x + band) * NE + e] = acc[i];
  }
}

// ---- forward: per-(b,c) solve ---------------------------------------------------------------------------
// In-place Cholesky of the D x D SPD matrix M (lower factor), then the inverse M^-1 = L^-T L^-1 into Minv.  One warp;
// Wk is D*D scratch.  Returns sum log(diag(L) + 1e-8) on every lane.
__device__ double rmi_chol_inv(double* M, double* Minv, double* Wk, int D, int lane) {
  if (lane == 0) {
    for (int j = 0; j < D; ++j) {
      double d = M[j * D + j];
      for (int k = 0; k < j; ++k) d -= M[j * D + k] * M[j * D + k];
      d = sqrt(d);
      M[j * D + j] = d;
      for (int i = j + 1; i < D; ++i) {
        double v = M[i * D + j];
        for (int k = 0; k < j; ++k) v -= M[i * D + k] * M[j * D + k];
        M[i * D + j] = v / d;
      }
    }
  }
  __syncwarp();
  if (lane < D) {                                            // column `lane` of L^-1 by forward substitution
    const int c = lane;
    for (int i = 0; i < D; ++i) {
      double v = i == c ? 1.0 : 0.0;
      for (int k = c; k < i; ++k) v -= M[i * D + k] * Wk[k * D + c];
      Wk[i * D + c] = i < c ? 0.0 : v / M[i * D + i];
    }
  }
  __syncwarp();
  for (int e = lane; e < D * D; e += 32) {
    const int i = e / D, j = e % D;
    double v = 0.0;
    for (int k = (i > j ? i : j); k < D; ++k) v += Wk[k * D + i] * Wk[k * D + j];
    Minv[e] = v;
  }
  double ld = 0.0;
  for (int j = 0; j < D; ++j) ld += log(M[j * D + j] + 1e-8);
  __syncwarp();
  return ld;
}

template <int R>
__global__ void __launch_bounds__(32)
k_rmi_solve(RmiArgs a, const double* __restrict__ part, int nbands, double* __restrict__ rmi_bc, double* __restrict__ g1,
            double* __restrict__ g2, double* __restrict__ mxy) {
  constexpr int D = R * R, NE = rmi_entries(R);
  __shared__ double Sm[NE];
  __shared__ double X[D * D], Pm[D * D], Q[D * D], Am[D * D], Wk[D * D], Inv[D * D];
  const int bc = blockIdx.x, lane = threadIdx.x;
  for (int e = lane; e < NE; e += 32) {
    double v = 0.0;
    for (int k = 0; k < nbands; ++k) v += part[((int64_t)bc * nbands + k) * NE + e];   // fixed order
    Sm[e] = v;
  }
  __syncwarp();
  const double n = (double)a.nY * (double)a.nX;
  const double* Sx = Sm; const double* Sy = Sm + D; const double* Sxy = Sm + 2 * D;
  const double* Sxx = Sxy + D * D; const double* Syy = Sxx + D * (D + 1) / 2;
  for (int e = lane; e < D * D; e += 32) {
    const int k = e / D, l = e % D, lo = k < l ? k : l, hi = k < l ? l : k;
    const int t = lo * D - lo * (lo - 1) / 2 + (hi - lo);
    X[e] = Sxx[t] - Sx[k] * Sx[l] / n;
    Pm[e] = Syy[t] - Sy[k] * Sy[l] / n + (k == l ? RMI_ALPHA : 0.0);
    Q[e] = Sxy[e] - Sx[k] * Sy[l] / n;
  }
  __syncwarp();
  rmi_chol_inv(Pm, Inv, Wk, D, lane);                         // Inv = P^-1
  for (int e = lane; e < D * D; e += 32) {                    // A = Q P^-1
    const int i = e / D, j = e % D;
    double v = 0.0;
    for (int k = 0; k < D; ++k) v += Q[i * D + k] * Inv[k * D + j];
    Am[e] = v;
  }
  __syncwarp();
  for (int e = lane; e < D * D; e += 32) {                    // M = X - A Q^T + alpha I   (into X)
    const int i = e / D, j = e % D;
    double v = 0.0;
    for (int k = 0; k < D; ++k) v += Am[i * D + k] * Q[j * D + k];
    X[e] = X[e] - v + (i == j ? RMI_ALPHA : 0.0);
  }
  __syncwarp();
  const double ld = rmi_chol_inv(X, Inv, Wk, D, lane);        // Inv = M^-1, ld = 0.5 * log det M (chol diagonal)
  const double coef = (double)a.lw * (double)a.wr / ((double)a.B * (double)D);
  for (int e = lane; e < D * D; e += 32) {                    // T = A^T M^-1 (into Pm)
    const int i = e / D, j = e % D;
    double v = 0.0;
    for (int k = 0; k < D; ++k) v += Am[k * D + i] * Inv[k * D + j];
    Pm[e] = v;
  }
  __syncwarp();
  for (int e = lane; e < D * D; e += 32) {                    // 2 dP = T A,  dQ^T = -T
    const int i = e / D, j = e % D;
    double v = 0.0;
    for (int k = 0; k < D; ++k) v += Pm[i * D + k] * Am[k * D + j];
    g1[(int64_t)bc * D * D + e] = coef * v;
    g2[(int64_t)bc * D * D + e] = -coef * Pm[e];
  }
  if (lane < D) {
    mxy[(int64_t)bc * 2 * D + lane] = Sx[lane] / n;
    mxy[(int64_t)bc * 2 * D + D + lane] = Sy[lane] / n;
  }
  if (lane == 0) rmi_bc[bc] = ld;
}

__global__ void __launch_bounds__(1024)
k_rmi_finalize(RmiArgs a, const float* __restrict__ part_bce, const int* __restrict__ part_cnt, int64_t n,
               const double* __restrict__ rmi_bc, double* __restrict__ fin, float* __restrict__ out) {
  block_sum2_1024<double, long long>(part_bce, part_cnt, n, [&](const double& ab, const long long& ac) {
    const double inv_n = 1.0 / ((double)ac + 1.0);
    double rmi = 0.0;
    for (int c = 0; c < a.K; ++c) {                           // sum_c mean_b(rmi_bc) / half_d
      double m = 0.0;
      for (int b = 0; b < a.B; ++b) m += rmi_bc[b * a.K + c];
      rmi += m / (double)a.B;
    }
    rmi /= (double)(a.r * a.r);
    const double loss = (double)a.lw * ((double)a.wb * ab * inv_n + (double)a.wr * rmi);
    fin[0] = loss;
    fin[1] = (double)a.lw * (double)a.wb * inv_n;             // d loss / d (sum of the BCE terms)
    fin[2] = rmi;
    fin[3] = (double)ac;
    out[0] = (float)loss;
  });
}

// ---- backward ----------------------------------------------------------------------------------------
template <int R>
__global__ void __launch_bounds__(256)
k_rmi_dpool(RmiArgs a, const float* __restrict__ P, const uint8_t* __restrict__ L, const double* __restrict__ g1,
            const double* __restrict__ g2, const double* __restrict__ mxy, const float* __restrict__ grad_out,
            float* __restrict__ dP) {
  constexpr int D = R * R;
  __shared__ double G1[D * D], G2[D * D], mx[D], my[D];
  const int bc = blockIdx.y;
  for (int e = threadIdx.x; e < D * D; e += 256) { G1[e] = g1[(int64_t)bc * D * D + e]; G2[e] = g2[(int64_t)bc * D * D + e]; }
  if (threadIdx.x < D) { mx[threadIdx.x] = mxy[(int64_t)bc * 2 * D + threadIdx.x]; my[threadIdx.x] = mxy[(int64_t)bc * 2 * D + D + threadIdx.x]; }
  __syncthreads();
  const int64_t HWp = (int64_t)a.Hp * a.Wp;
  const int64_t u = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (u >= HWp) return;
  const int uy = (int)(u / a.Wp), ux = (int)(u - (int64_t)uy * a.Wp);
  const float* Pb = P + (int64_t)bc * HWp;
  const uint8_t* Lb = L + (int64_t)bc * HWp;
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < D; ++k) {
    const int jy = uy - k / R, jx = ux - k % R;               // point whose neighbour k is this pooled pixel
    if (jy < 0 || jx < 0 || jy >= a.nY || jx >= a.nX) continue;
    double v = 0.0;
#pragma unroll
    for (int l = 0; l < D; ++l) {
      const int64_t o = (int64_t)(jy + l / R) * a.Wp + jx + l % R;
      v += G1[k * D + l] * ((double)Pb[o] - my[l]) + G2[k * D + l] * ((double)rmi_label_value(Lb[o], a.way, a.s) - mx[l]);
    }
    acc += v;
  }
  dP[(int64_t)bc * HWp + u] = (float)(acc * (grad_out ? (double)grad_out[0] : 1.0));
}

__global__ void __launch_bounds__(BT * BTY)
k_rmi_bwd_tile(RmiArgs a, const float* __restrict__ dP, const uint8_t* __restrict__ Am, const double* __restrict__ fin,
               const float* __restrict__ grad_out, float* __restrict__ dseg, int kc, int pitch) {
  const int tx = threadIdx.x & (BT - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int x = blockIdx.x * BT + tx, y = blockIdx.y * BTY + ty;
  const int64_t HWo = (int64_t)a.H * a.W, HWp = (int64_t)a.Hp * a.Wp;
  const float cb = (float)fin[1] * (grad_out ? grad_out[0] : 1.f);
  int tv = -1;
  int64_t u = -1;                                  // pooled pixel whose window holds this label pixel
  int slot = 0;
  if (x < a.W && y < a.H) {
    int64_t t = a.target[(int64_t)b * HWo + (int64_t)y * a.W + x];
    if (t < 0) t = 255;
    tv = t < a.K ? (int)t : -1;
    const int uy = (y + a.pad) / a.s, ux = (x + a.pad) / a.s;
    if (uy < a.Hp && ux < a.Wp) {
      u = (int64_t)uy * a.Wp + ux;
      slot = (y + a.pad - uy * a.s) * a.s + (x + a.pad - ux * a.s);
    }
  }
  const float inv_s2 = 1.f / (float)(a.s * a.s);
  up_bwd_tile(a, a.seg, dseg, kc, pitch, [](const UpTile&, const UpPix&, float*) {},
              [&](int c0, int cn, const UpPix& px, const float* S, float* G) {
    const float ly = px.ly, lx = px.lx;
    for (int cc = 0; cc < cn; ++cc) {
      float gv = 0.f;
      if (tv >= 0) {
        const int c = c0 + cc;
        const float* p = S + cc * pitch;
        // the nested form of k_rmi_pool: its FMA chain, so the forward and backward see the same z
        const float z = (1.f - ly) * ((1.f - lx) * p[px.i00] + lx * p[px.i01]) +
                        ly * ((1.f - lx) * p[px.i10] + lx * p[px.i11]);
        const float sg = 1.f / (1.f + expf(-z));
        gv = cb * (sg - (tv == c ? 1.f : 0.f));                                  // BCE with logits
        if (u >= 0) {
          const int64_t o = ((int64_t)b * a.K + c) * HWp + u;
          const float dp = a.way == 0 ? (Am[o] == slot ? dP[o] : 0.f) : dP[o] * inv_s2;
          gv += dp * sg * (1.f - sg);
        }
      }
      G[((size_t)cc * BTY + ty) * BT + tx] = gv;
    }
  });
}

}  // namespace pcl

using namespace pcl;

namespace {

struct RmiLayout {
  size_t P, L, A, dP, bce, cnt, part, rmi, g1, g2, mxy, fin, total;
  int64_t pool_blocks;
  int nbands;
};

// Validates the geometry and parameters; fills the pooled-map sizes.  Refuses (PCL_ERR_UNSUPPORTED) what the reference
// accepts but the engine does not implement: radius 5-10, pool way 2, stride > 4, down-sampling, a pooled map smaller
// than the radius, more than 256 classes.
int rmi_geometry(int B, int K, int h, int w, int H, int W, int radius, int way, int stride, RmiArgs* a) {
  const int st = up_geometry(B, K, h, w, H, W, a);
  if (st != PCL_OK) return st;
  if (radius < 1 || radius > 10 || way < 0 || way > 3 || stride < 1) return PCL_ERR_ARG;
  if (radius > RMI_R_MAX || way > 1 || stride > RMI_S_MAX || K > 256 || H < h || W < w) return PCL_ERR_UNSUPPORTED;
  a->r = radius; a->way = way; a->s = stride; a->pad = stride / 2;
  a->Hp = (H + 2 * a->pad - stride) / stride + 1;
  a->Wp = (W + 2 * a->pad - stride) / stride + 1;
  if (a->Hp < radius || a->Wp < radius) return PCL_ERR_UNSUPPORTED;
  a->nY = a->Hp - radius + 1; a->nX = a->Wp - radius + 1;
  return PCL_OK;
}

RmiLayout rmi_layout(const RmiArgs& a) {
  RmiLayout l;
  const int64_t n = (int64_t)a.B * a.K * a.Hp * a.Wp, BK = (int64_t)a.B * a.K;
  const int D = a.r * a.r;
  l.pool_blocks = (int64_t)ceil_div(a.Wp, PT_X) * ceil_div(a.Hp, PT_Y) * a.B;
  l.nbands = ceil_div(a.nY, MB_Y);
  size_t o = 0;
  l.P = o;    o = align256(o + n * sizeof(float));
  l.dP = o;   o = align256(o + n * sizeof(float));
  l.L = o;    o = align256(o + n);
  l.A = o;    o = align256(o + n);
  l.bce = o;  o = align256(o + l.pool_blocks * sizeof(float));
  l.cnt = o;  o = align256(o + l.pool_blocks * sizeof(int));
  l.part = o; o = align256(o + (size_t)BK * l.nbands * rmi_entries(a.r) * sizeof(double));
  l.rmi = o;  o = align256(o + BK * sizeof(double));
  l.g1 = o;   o = align256(o + BK * D * D * sizeof(double));
  l.g2 = o;   o = align256(o + BK * D * D * sizeof(double));
  l.mxy = o;  o = align256(o + BK * 2 * D * sizeof(double));
  l.fin = o;  o = align256(o + 4 * sizeof(double));
  l.total = o;
  return l;
}

int rmi_make(const float* seg, const int64_t* target, int B, int K, int h, int w, int H, int W, int radius, int way,
             int stride, float weight_lambda, int lambda_way, float loss_weight, RmiArgs* a) {
  if (!seg || !target) return PCL_ERR_ARG;
  const int st = rmi_geometry(B, K, h, w, H, W, radius, way, stride, a);
  if (st != PCL_OK) return st;
  a->seg = seg; a->target = target;
  a->lw = loss_weight;
  a->wb = lambda_way ? weight_lambda : 1.f;
  a->wr = lambda_way ? 1.f - weight_lambda : weight_lambda;
  return PCL_OK;
}

template <int R>
int rmi_moments_solve(const RmiArgs& a, const RmiLayout& l, char* sc, cudaStream_t s) {
  k_rmi_moments<R><<<dim3((unsigned)l.nbands, (unsigned)(a.B * a.K)), 256, 0, s>>>(
      a, (const float*)(sc + l.P), (const uint8_t*)(sc + l.L), (double*)(sc + l.part));
  PCL_LAUNCH_CHECK();
  k_rmi_solve<R><<<a.B * a.K, 32, 0, s>>>(a, (const double*)(sc + l.part), l.nbands, (double*)(sc + l.rmi),
                                          (double*)(sc + l.g1), (double*)(sc + l.g2), (double*)(sc + l.mxy));
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

template <int R>
int rmi_dpool(const RmiArgs& a, const RmiLayout& l, const char* sc, const float* grad_loss, cudaStream_t s) {
  const int64_t HWp = (int64_t)a.Hp * a.Wp;
  k_rmi_dpool<R><<<dim3((unsigned)ceil_div64(HWp, 256), (unsigned)(a.B * a.K)), 256, 0, s>>>(
      a, (const float*)(sc + l.P), (const uint8_t*)(sc + l.L), (const double*)(sc + l.g1), (const double*)(sc + l.g2),
      (const double*)(sc + l.mxy), grad_loss, (float*)(sc + l.dP));
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

}  // namespace

extern "C" int64_t pcl_rmi_scratch_bytes(int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg, int32_t Wimg,
                                         int32_t radius, int32_t pool_way, int32_t pool_stride) {
  RmiArgs a;
  const int st = rmi_geometry(B, K, h, w, Himg, Wimg, radius, pool_way, pool_stride, &a);
  if (st != PCL_OK) return st;
  return (int64_t)rmi_layout(a).total;
}

extern "C" int pcl_rmi_fwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w,
                           int32_t Himg, int32_t Wimg, int32_t radius, int32_t pool_way, int32_t pool_stride,
                           float weight_lambda, int32_t lambda_way, float loss_weight, void* scratch, float* loss,
                           void* stream) {
  RmiArgs a;
  const int st = rmi_make(seg, target, B, K, h, w, Himg, Wimg, radius, pool_way, pool_stride, weight_lambda, lambda_way,
                          loss_weight, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && loss);
  cudaStream_t s = (cudaStream_t)stream;
  const RmiLayout l = rmi_layout(a);
  char* sc = (char*)scratch;
  // source patch of a pool tile: label rows / columns of REG_ROWS x REG_COLS at most, after its label region
  UpPlan pl;
  int rc = up_fwd_plan(a, up_patch_pitch(a, REG_ROWS, REG_COLS), (size_t)REG_ROWS * REG_COLS * sizeof(short), &pl);
  if (rc != PCL_OK) return rc;
  PCL_SMEM_OPT_IN(k_rmi_pool, 200 * 1024);
  k_rmi_pool<<<dim3((unsigned)ceil_div(a.Wp, PT_X), (unsigned)ceil_div(a.Hp, PT_Y), B), PT_X * PT_Y, pl.smem, s>>>(
      a, (float*)(sc + l.P), (uint8_t*)(sc + l.L), (uint8_t*)(sc + l.A), (float*)(sc + l.bce), (int*)(sc + l.cnt),
      pl.pitch, pl.kc);
  PCL_LAUNCH_CHECK();
  switch (radius) {
    case 1: rc = rmi_moments_solve<1>(a, l, sc, s); break;
    case 2: rc = rmi_moments_solve<2>(a, l, sc, s); break;
    case 3: rc = rmi_moments_solve<3>(a, l, sc, s); break;
    default: rc = rmi_moments_solve<4>(a, l, sc, s); break;
  }
  if (rc != PCL_OK) return rc;
  k_rmi_finalize<<<1, 1024, 0, s>>>(a, (const float*)(sc + l.bce), (const int*)(sc + l.cnt), l.pool_blocks,
                                    (const double*)(sc + l.rmi), (double*)(sc + l.fin), loss);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_rmi_bwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w,
                           int32_t Himg, int32_t Wimg, int32_t radius, int32_t pool_way, int32_t pool_stride,
                           float weight_lambda, int32_t lambda_way, float loss_weight, void* scratch,
                           const float* grad_loss, float* dseg, void* stream) {
  RmiArgs a;
  const int st = rmi_make(seg, target, B, K, h, w, Himg, Wimg, radius, pool_way, pool_stride, weight_lambda, lambda_way,
                          loss_weight, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && dseg);
  cudaStream_t s = (cudaStream_t)stream;
  const RmiLayout l = rmi_layout(a);
  char* sc = (char*)scratch;
  int rc = PCL_OK;
  switch (radius) {
    case 1: rc = rmi_dpool<1>(a, l, sc, grad_loss, s); break;
    case 2: rc = rmi_dpool<2>(a, l, sc, grad_loss, s); break;
    case 3: rc = rmi_dpool<3>(a, l, sc, grad_loss, s); break;
    default: rc = rmi_dpool<4>(a, l, sc, grad_loss, s); break;
  }
  if (rc != PCL_OK) return rc;
  return up_bwd_launch<k_rmi_bwd_tile>(a, s, dseg, (const float*)(sc + l.dP), (const uint8_t*)(sc + l.A),
                                       (const double*)(sc + l.fin), grad_loss);
}

// ==================================================================================================================
// Fused Lovasz-softmax segmentation loss of the contrast wrappers (FSCELOVASZLoss, lib/loss/loss_helper.py:77-124,
// built by lib/loss/loss_contrast_mem.py:187-194 with contrast.use_lovasz): replaces
//   F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True) + softmax + flatten_probas + lovasz_softmax_flat(
//   only_present=True)  (lib/loss/lovasz_loss.py:216-267)
// and its autograd backward without materialising the (B,K,Himg,Wimg) up-sampled logits, their softmax, the permuted
// copy or the masked gather, and without a host sync per class.  N = B*Himg*Wimg label pixels, q = (b*Himg + y)*Wimg + x.
//   k_lov_keys      tile kernel (pcl_upsample.cuh geometry): bilinear logits, softmax, per class the key
//                   d = bits(1.0f) - bits(e), e = |fg - p_c| (e in [0, 1]: the bit order is the value order, so an
//                   ascending sort of d is a descending sort of e); an ignored pixel gets LOV_SENT, which sorts last.
//                   Also the pixel's (max, sum of exp) for the backward and a u8 label copy.
//   sort            per class, stable LSD radix sort of (d, q) in 4 passes of 8 bits, classes in chunks chosen from the
//                   shapes.  Each pass: k_lov_hist (per-tile digit counts), k_lov_scan (exclusive scan per class, fixed
//                   order), k_lov_scatter (stable in-tile rank by warp ballots).  No CTA waits on another: the result
//                   does not depend on scheduling.  Ties in e keep ascending q (the input order).
//   k_lov_fgcount   fg count per tile of the sorted order, scanned by k_lov_scan (the class's gts is its total)
//   k_lov_loss      per sorted position i with cumfg F and cumbg i-F before it (exact integers): I = gts - F,
//                   U = gts + i - F, g = 1/U for a fg step, I/(U(U+1)) for a bg step (the reference's J_i - J_{i-1} in
//                   closed form, free of its fp32 cancellation); loss_c partials sum e*g in fp64, g is scattered to ge[c][q]
//   k_lov_finalize  mean of loss_c over the present classes (gts > 0), in a fixed order: the loss is bit-reproducible
//   k_lov_bwd_tile  recomputes p from the staged patch; dp_c = grad * ge_c * sgn(p_c - fg_c) / n_present, dz = p (dp - <p, dp>),
//                   then the transposed bilinear map into dseg (up_tile_flush: <= 4-way fp32 atomics, dseg reproducible to
//                   the last ulp or two)
// First-order HBM bytes at B=8, K=19, 128x256 -> 512x1024 (N = 4.19 M, K*N = 79.7 M keys): the keys kernel writes 318 MB;
// each sort pass reads the keys twice and the payload once and writes both (~20 B per key, 1.6 GB per pass); the loss
// reads the sorted pairs twice and scatters ge (~1 GB); the backward reads ge (318 MB) and seg, and writes dseg (DESIGN §4).
namespace pcl {

constexpr uint32_t LOV_ONE = 0x3F800000u;     // bits of 1.0f
constexpr uint32_t LOV_SENT = 0x3FFFFFFFu;    // ignored pixel: above every d = LOV_ONE - bits(e) <= LOV_ONE
constexpr int LOV_THREADS = 256;
constexpr int LOV_ITEMS = 8;
constexpr int LOV_TILE = LOV_THREADS * LOV_ITEMS;   // keys per sort / loss tile
constexpr int LOV_RADIX = 256;
constexpr int LOV_PASSES = 4;                       // 4 x 8 bits cover the 30 live bits of d

struct LovArgs : UpGeom {
  const float* seg; const int64_t* target;
  int ignore_index;
  int64_t N;                    // B*H*W
};

// the label of pixel (b, y, x) if it counts (not ignore_index, inside [0, K)), else -1
__device__ __forceinline__ int lov_label(const LovArgs& a, int64_t q) {
  const int64_t t = a.target[q];
  return (t != (int64_t)a.ignore_index && t >= 0 && t < a.K) ? (int)t : -1;
}

// ---- keys --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BT * BTY)
k_lov_keys(LovArgs a, uint32_t* __restrict__ keys, float2* __restrict__ ms, uint8_t* __restrict__ lab, int pitch, int kc) {
  extern __shared__ float sm[];                    // [kc][pitch] source patch
  __shared__ int s_y0[BTY], s_y1[BTY], s_x0[BT], s_x1[BT];
  __shared__ float s_ly[BTY], s_lx[BT];
  const int tx = threadIdx.x & (BT - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int X0 = blockIdx.x * BT, Y0 = blockIdx.y * BTY;
  const int x = X0 + tx, y = Y0 + ty;
  const UpTile g = up_tile_coords(X0, Y0, a.H, a.W, a.h, a.w, a.ry, a.rx, s_y0, s_y1, s_ly, s_x0, s_x1, s_lx);
  const UpPix px = up_pix(g, tx, ty, s_y0, s_y1, s_ly, s_x0, s_x1, s_lx);
  const bool inside = x < a.W && y < a.H;
  const int64_t q = ((int64_t)b * a.H + y) * a.W + x;
  const int t = inside ? lov_label(a, q) : -1;
  float m = -CUDART_INF_F, se = 0.f;
  const bool one = a.K <= kc;                      // one staged chunk: the second sweep reuses it
  for (int c0 = 0; c0 < a.K; c0 += kc) {
    const int cn = min(kc, a.K - c0);
    up_stage(a, a.seg, b, c0, cn, g.ys_base, g.xs_base, g.ys_n, g.xs_n, pitch, sm);
    __syncthreads();
    for (int cc = 0; cc < cn; ++cc) {
      const float v = up_logit(px, sm + cc * pitch);
      if (v > m) { se = se * __expf(m - v) + 1.f; m = v; }     // online sum of exp
      else       { se += __expf(v - m); }
    }
    if (!one) __syncthreads();
  }
  if (inside) {
    ms[q] = make_float2(m, se);
    lab[q] = (uint8_t)(t >= 0 ? t : 0);
  }
  for (int c0 = 0; c0 < a.K; c0 += kc) {
    const int cn = min(kc, a.K - c0);
    if (!one) {
      up_stage(a, a.seg, b, c0, cn, g.ys_base, g.xs_base, g.ys_n, g.xs_n, pitch, sm);
      __syncthreads();
    }
    if (inside) {
      for (int cc = 0; cc < cn; ++cc) {
        const int c = c0 + cc;
        uint32_t d = LOV_SENT;
        if (t >= 0) {
          const float p = __expf(up_logit(px, sm + cc * pitch) - m) / se;
          const float e = fabsf((t == c ? 1.f : 0.f) - p);
          d = LOV_ONE - __float_as_uint(e);
        }
        keys[(int64_t)c * a.N + q] = d;
      }
    }
    if (!one) __syncthreads();
  }
}

// ---- sort ----------------------------------------------------------------------------------------------
// hist[c][digit][tile]: digit counts of each tile (shared-memory atomics: integer counts, order-free)
__global__ void __launch_bounds__(LOV_THREADS)
k_lov_hist(const uint32_t* __restrict__ keys, int64_t N, int shift, int ntiles, int* __restrict__ hist) {
  __shared__ int s_h[LOV_RADIX];
  const int c = blockIdx.y;
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t* k = keys + (int64_t)c * N;
  const int64_t base = (int64_t)blockIdx.x * LOV_TILE;
  for (int r = 0; r < LOV_ITEMS; ++r) {
    const int64_t i = base + r * LOV_THREADS + threadIdx.x;
    if (i < N) atomicAdd(&s_h[(k[i] >> shift) & (LOV_RADIX - 1)], 1);
  }
  __syncthreads();
  hist[((int64_t)c * LOV_RADIX + threadIdx.x) * ntiles + blockIdx.x] = s_h[threadIdx.x];
}

// In-place exclusive scan of len ints per class (blockIdx.x = class, row stride `stride`); the total goes to total[c]
// when total is given.  One CTA per class, sequential over chunks: a fixed order, no inter-CTA dependency.
__global__ void __launch_bounds__(1024)
k_lov_scan(int* __restrict__ data, int64_t len, int64_t stride, int* __restrict__ total) {
  __shared__ int s_w[32];
  int* d = data + (int64_t)blockIdx.x * stride;
  int carry = 0;
  for (int64_t base = 0; base < len; base += 4 * 1024) {
    int v[4], s = 0;
    const int64_t i0 = base + 4 * (int64_t)threadIdx.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) { v[j] = i0 + j < len ? d[i0 + j] : 0; s += v[j]; }
    const int excl = block_exclusive_scan_1024(s, s_w);
    int run = carry + excl;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (i0 + j < len) d[i0 + j] = run;
      run += v[j];
    }
    __syncthreads();
    if (threadIdx.x == 1023) s_w[0] = excl + s;                   // chunk total: the last thread's inclusive sum
    __syncthreads();
    carry += s_w[0];
    __syncthreads();
  }
  if (total && threadIdx.x == 0) total[blockIdx.x] = carry;
}

// One stable LSD pass: keys_in / vals_in (vals_in null on the first pass: the payload is the index q) -> keys_out /
// vals_out at offs[c][digit][tile] + the item's rank among the tile's items of its digit.  Items go in index order: round
// r, warp w, lane l holds index r*256 + 32 w + l; within a warp the peers of a digit come from 8 ballots.
__global__ void __launch_bounds__(LOV_THREADS)
k_lov_scatter(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in, int64_t N, int shift,
              int ntiles, const int* __restrict__ offs, uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out) {
  __shared__ int s_cnt[2 * LOV_RADIX * (LOV_THREADS / 32)];         // [buffer][digit][warp]
  __shared__ int s_base[LOV_RADIX];                                  // global offset of the tile's digit + running count
  const int c = blockIdx.y;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  constexpr int NW = LOV_THREADS / 32;
  const int64_t cN = (int64_t)c * N;
  for (int i = threadIdx.x; i < 2 * LOV_RADIX * NW; i += LOV_THREADS) s_cnt[i] = 0;
  s_base[threadIdx.x] = offs[((int64_t)c * LOV_RADIX + threadIdx.x) * ntiles + blockIdx.x];
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * LOV_TILE;
  const unsigned lt = (1u << lane) - 1u;
  for (int r = 0; r < LOV_ITEMS; ++r) {
    int* cnt = s_cnt + (r & 1) * LOV_RADIX * NW;
    const int64_t i = base + r * LOV_THREADS + threadIdx.x;
    const bool valid = i < N;
    uint32_t key = 0, val = 0;
    if (valid) {
      key = keys_in[cN + i];
      val = vals_in ? vals_in[cN + i] : (uint32_t)i;
    }
    const int dg = (int)((key >> shift) & (LOV_RADIX - 1));
    unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int bit = 0; bit < 8; ++bit) {
      const int on = (dg >> bit) & 1;
      const unsigned bb = __ballot_sync(0xffffffffu, on);
      peers &= on ? bb : ~bb;
    }
    const int rank = __popc(peers & lt);
    if (valid && rank == 0) cnt[dg * NW + wid] = __popc(peers);
    __syncthreads();
    {                                                                // thread = digit: warp counts -> offsets
      int* row = cnt + threadIdx.x * NW;
      int run = s_base[threadIdx.x];
#pragma unroll
      for (int w = 0; w < NW; ++w) { const int n = row[w]; row[w] = run; run += n; }
      s_base[threadIdx.x] = run;
      int* nxt = s_cnt + ((r + 1) & 1) * LOV_RADIX * NW + threadIdx.x * NW;
#pragma unroll
      for (int w = 0; w < NW; ++w) nxt[w] = 0;
    }
    __syncthreads();
    if (valid) {
      const int64_t o = cN + cnt[dg * NW + wid] + rank;
      keys_out[o] = key;
      vals_out[o] = val;
    }
  }
}

// ---- scan and loss -----------------------------------------------------------------------------------------
__device__ __forceinline__ bool lov_fg(uint32_t key, uint32_t q, const uint8_t* lab, int c) {
  return key != LOV_SENT && (int)lab[q] == c;
}

__global__ void __launch_bounds__(LOV_THREADS)
k_lov_fgcount(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint8_t* __restrict__ lab,
              int64_t N, int c0, int ntiles, int* __restrict__ tilefg) {
  __shared__ int s_w[LOV_THREADS / 32];
  const int c = blockIdx.y;
  const int64_t cN = (int64_t)c * N;
  const int64_t base = (int64_t)blockIdx.x * LOV_TILE;
  int n = 0;
  for (int r = 0; r < LOV_ITEMS; ++r) {
    const int64_t i = base + r * LOV_THREADS + threadIdx.x;
    if (i < N) n += lov_fg(keys[cN + i], vals[cN + i], lab, c0 + c);
  }
  n = warp_sum_i(n);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < LOV_THREADS / 32; ++w) s += s_w[w];
    tilefg[(int64_t)(c0 + c) * ntiles + blockIdx.x] = s;
  }
}

// Thread t of a tile owns the LOV_ITEMS consecutive sorted positions base + t*LOV_ITEMS + j.
__global__ void __launch_bounds__(LOV_THREADS)
k_lov_loss(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint8_t* __restrict__ lab,
           int64_t N, int c0, int ntiles, const int* __restrict__ tilefg, const int* __restrict__ gts_all,
           float* __restrict__ ge, double* __restrict__ part) {
  __shared__ int s_w[LOV_THREADS / 32];
  __shared__ double s_d[LOV_THREADS / 32];
  const int c = blockIdx.y, cg = c0 + c;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t cN = (int64_t)c * N;
  const int64_t i0 = (int64_t)blockIdx.x * LOV_TILE + (int64_t)threadIdx.x * LOV_ITEMS;
  const int64_t gts = gts_all[cg];
  float* gec = ge + (int64_t)cg * N;
  uint32_t key[LOV_ITEMS], q[LOV_ITEMS];
  int nfg = 0;
#pragma unroll
  for (int j = 0; j < LOV_ITEMS; ++j) {
    key[j] = LOV_SENT; q[j] = 0;
    if (i0 + j < N) { key[j] = keys[cN + i0 + j]; q[j] = vals[cN + i0 + j]; }
    nfg += lov_fg(key[j], q[j], lab, cg);
  }
  int incl = nfg;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  int wbase = 0;
  for (int w = 0; w < wid; ++w) wbase += s_w[w];
  int64_t F = (int64_t)tilefg[(int64_t)cg * ntiles + blockIdx.x] + wbase + incl - nfg;   // fg before position i0
  double acc = 0.0;
#pragma unroll
  for (int j = 0; j < LOV_ITEMS; ++j) {
    const int64_t i = i0 + j;
    if (i >= N) break;
    if (key[j] == LOV_SENT || gts == 0) { gec[q[j]] = 0.f; continue; }
    const bool fg = (int)lab[q[j]] == cg;
    const double I = (double)(gts - F), U = (double)(gts + (i - F));
    const double gv = fg ? 1.0 / U : I / (U * (U + 1.0));
    acc += (double)__uint_as_float(LOV_ONE - key[j]) * gv;
    gec[q[j]] = (float)gv;
    F += fg;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) s_d[wid] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < LOV_THREADS / 32; ++w) s += s_d[w];                      // fixed order
    part[(int64_t)cg * ntiles + blockIdx.x] = s;
  }
}

// loss = sum over present classes of loss_c / n_present (0 when no pixel counts); fin = {loss, n_present}
__global__ void __launch_bounds__(256)
k_lov_finalize(const double* __restrict__ part, const int* __restrict__ gts, int K, int ntiles, float* __restrict__ fin,
               float* __restrict__ out) {
  __shared__ double s_d[256];
  double tot = 0.0;
  int npres = 0;
  for (int c = 0; c < K; ++c) {
    double s = 0.0;
    for (int t = threadIdx.x; t < ntiles; t += 256) s += part[(int64_t)c * ntiles + t];
    s_d[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) s_d[threadIdx.x] += s_d[threadIdx.x + o];
      __syncthreads();
    }
    if (gts[c] > 0) { tot += s_d[0]; ++npres; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float loss = npres ? (float)(tot / (double)npres) : 0.f;
    fin[0] = loss;
    fin[1] = (float)npres;
    out[0] = loss;
  }
}

// ---- backward ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BT * BTY, 4)     // 4 CTAs per SM: 64 registers, no spill
k_lov_bwd_tile(LovArgs a, const float2* __restrict__ ms, const float* __restrict__ ge, const float* __restrict__ fin,
               const float* __restrict__ grad_out, float* __restrict__ dseg, int kc, int pitch) {
  const int tx = threadIdx.x & (BT - 1), ty = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int x = blockIdx.x * BT + tx, y = blockIdx.y * BTY + ty;
  const int64_t q = ((int64_t)b * a.H + y) * a.W + x;
  const float npres = fin[1];
  const float scale = npres > 0.f ? (grad_out ? grad_out[0] : 1.f) / npres : 0.f;
  int t = -1;
  float m = 0.f, se = 1.f;
  if (x < a.W && y < a.H) {
    t = lov_label(a, q);
    const float2 v = ms[q];
    m = v.x; se = v.y;
  }
  const bool one = a.K <= kc;
  float dot = 0.f;                                 // <p, dp>
  up_bwd_tile(a, a.seg, dseg, kc, pitch, [&](const UpTile& g, const UpPix& px, float* S) {
    if (one) return;                               // several chunks: <p, dp> first
    for (int c0 = 0; c0 < a.K; c0 += kc) {
      const int cn = min(kc, a.K - c0);
      __syncthreads();
      up_stage(a, a.seg, b, c0, cn, g.ys_base, g.xs_base, g.ys_n, g.xs_n, pitch, S);
      __syncthreads();
      if (t >= 0) {
        for (int cc = 0; cc < cn; ++cc) {
          const int c = c0 + cc;
          const float p = __expf(up_logit(px, S + cc * pitch) - m) / se;
          const float f = t == c ? 1.f : 0.f;
          const float dp = p > f ? ge[(int64_t)c * a.N + q] : (p < f ? -ge[(int64_t)c * a.N + q] : 0.f);
          dot += p * dp;
        }
      }
    }
  }, [&](int c0, int cn, const UpPix& px, const float* S, float* G) {
    for (int cc = 0; cc < cn; ++cc) {              // dp (and <p, dp> when one chunk holds every class)
      float dp = 0.f;
      if (t >= 0) {
        const int c = c0 + cc;
        const float p = __expf(up_logit(px, S + cc * pitch) - m) / se;
        const float f = t == c ? 1.f : 0.f;
        dp = p > f ? ge[(int64_t)c * a.N + q] : (p < f ? -ge[(int64_t)c * a.N + q] : 0.f);
        if (one) dot += p * dp;
      }
      G[((size_t)cc * BTY + ty) * BT + tx] = dp;
    }
    for (int cc = 0; cc < cn; ++cc) {              // dz = scale * p (dp - <p, dp>)
      float gv = 0.f;
      if (t >= 0) {
        const float p = __expf(up_logit(px, S + cc * pitch) - m) / se;
        gv = scale * p * (G[((size_t)cc * BTY + ty) * BT + tx] - dot);
      }
      G[((size_t)cc * BTY + ty) * BT + tx] = gv;
    }
  });
}

}  // namespace pcl

using namespace pcl;

namespace {

struct LovLayout {
  size_t keys, vals, keys2, vals2, ge, ms, lab, hist, tilefg, gts, part, fin, total;
  int ntiles, cc;
};

// Geometry of the losses that sort or select over the label pixels (Lovasz, OHEM): refuses (PCL_ERR_UNSUPPORTED) a label
// grid smaller than the logits, more than 256 classes and N = B*H*W >= 2^31 (pixel indices are 32-bit).
int sort_geometry(int B, int K, int h, int w, int H, int W, UpGeom* g) {
  const int st = up_geometry(B, K, h, w, H, W, g);
  if (st != PCL_OK) return st;
  if (H < h || W < w || K > 256) return PCL_ERR_UNSUPPORTED;
  if ((int64_t)B * H * W >= ((int64_t)1 << 31)) return PCL_ERR_UNSUPPORTED;
  return PCL_OK;
}

int lov_geometry(int B, int K, int h, int w, int H, int W, LovArgs* a) {
  const int st = sort_geometry(B, K, h, w, H, W, a);
  a->N = (int64_t)B * H * W;
  return st;
}

// Classes sorted together: a quarter of them (rounded up), so the sort's three extra key / payload buffers stay at
// about 3/4 of the keys buffer.
LovLayout lov_layout(const LovArgs& a) {
  LovLayout l;
  l.ntiles = (int)ceil_div64(a.N, LOV_TILE);
  l.cc = (a.K + 3) / 4;
  const size_t kn = (size_t)a.K * a.N, cn = (size_t)l.cc * a.N;
  size_t o = 0;
  l.keys = o;   o = align256(o + kn * 4);
  l.ge = o;     o = align256(o + kn * 4);
  l.vals = o;   o = align256(o + cn * 4);
  l.keys2 = o;  o = align256(o + cn * 4);
  l.vals2 = o;  o = align256(o + cn * 4);
  l.ms = o;     o = align256(o + (size_t)a.N * 8);
  l.lab = o;    o = align256(o + (size_t)a.N);
  l.hist = o;   o = align256(o + (size_t)l.cc * LOV_RADIX * l.ntiles * 4);
  l.tilefg = o; o = align256(o + (size_t)a.K * l.ntiles * 4);
  l.gts = o;    o = align256(o + (size_t)a.K * 4);
  l.part = o;   o = align256(o + (size_t)a.K * l.ntiles * 8);
  l.fin = o;    o = align256(o + 4 * sizeof(float));
  l.total = o;
  return l;
}

int lov_make(const float* seg, const int64_t* target, int B, int K, int h, int w, int H, int W, int ignore_index,
             LovArgs* a) {
  if (!seg || !target) return PCL_ERR_ARG;
  const int st = lov_geometry(B, K, h, w, H, W, a);
  if (st != PCL_OK) return st;
  a->seg = seg; a->target = target; a->ignore_index = ignore_index;
  return PCL_OK;
}

}  // namespace

extern "C" int64_t pcl_lovasz_scratch_bytes(int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg, int32_t Wimg) {
  LovArgs a;
  const int st = lov_geometry(B, K, h, w, Himg, Wimg, &a);
  if (st != PCL_OK) return st;
  return (int64_t)lov_layout(a).total;
}

extern "C" int pcl_lovasz_fwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w,
                              int32_t Himg, int32_t Wimg, int32_t ignore_index, void* scratch, float* loss, void* stream) {
  LovArgs a;
  const int st = lov_make(seg, target, B, K, h, w, Himg, Wimg, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && loss);
  cudaStream_t s = (cudaStream_t)stream;
  const LovLayout l = lov_layout(a);
  char* sc = (char*)scratch;
  uint32_t* keys = (uint32_t*)(sc + l.keys);
  uint32_t* vals = (uint32_t*)(sc + l.vals);
  uint32_t* keys2 = (uint32_t*)(sc + l.keys2);
  uint32_t* vals2 = (uint32_t*)(sc + l.vals2);
  const uint8_t* lab = (const uint8_t*)(sc + l.lab);
  int* hist = (int*)(sc + l.hist);
  int* tilefg = (int*)(sc + l.tilefg);
  int* gts = (int*)(sc + l.gts);
  UpPlan pl;
  const int rc = up_fwd_plan(a, up_patch_pitch(a, BTY, BT), 0, &pl);
  if (rc != PCL_OK) return rc;
  PCL_SMEM_OPT_IN(k_lov_keys, 200 * 1024);
  k_lov_keys<<<dim3((unsigned)ceil_div(Wimg, BT), (unsigned)ceil_div(Himg, BTY), B), BT * BTY, pl.smem, s>>>(
      a, keys, (float2*)(sc + l.ms), (uint8_t*)(sc + l.lab), pl.pitch, pl.kc);
  PCL_LAUNCH_CHECK();
  const int nt = l.ntiles;
  for (int c0 = 0; c0 < K; c0 += l.cc) {
    const int cn = min(l.cc, K - c0);
    uint32_t* kA = keys + (int64_t)c0 * a.N;
    const dim3 grid((unsigned)nt, (unsigned)cn);
    for (int p = 0; p < LOV_PASSES; ++p) {               // A -> B -> A -> B -> A
      const uint32_t* kin = p & 1 ? keys2 : kA;
      const uint32_t* vin = p == 0 ? nullptr : (p & 1 ? vals2 : vals);
      uint32_t* kout = p & 1 ? kA : keys2;
      uint32_t* vout = p & 1 ? vals : vals2;
      k_lov_hist<<<grid, LOV_THREADS, 0, s>>>(kin, a.N, 8 * p, nt, hist);
      PCL_LAUNCH_CHECK();
      k_lov_scan<<<cn, 1024, 0, s>>>(hist, (int64_t)LOV_RADIX * nt, (int64_t)LOV_RADIX * nt, nullptr);
      PCL_LAUNCH_CHECK();
      k_lov_scatter<<<grid, LOV_THREADS, 0, s>>>(kin, vin, a.N, 8 * p, nt, hist, kout, vout);
      PCL_LAUNCH_CHECK();
    }
    k_lov_fgcount<<<grid, LOV_THREADS, 0, s>>>(kA, vals, lab, a.N, c0, nt, tilefg);
    PCL_LAUNCH_CHECK();
    k_lov_scan<<<cn, 1024, 0, s>>>(tilefg + (int64_t)c0 * nt, nt, nt, gts + c0);
    PCL_LAUNCH_CHECK();
    k_lov_loss<<<grid, LOV_THREADS, 0, s>>>(kA, vals, lab, a.N, c0, nt, tilefg, gts, (float*)(sc + l.ge),
                                            (double*)(sc + l.part));
    PCL_LAUNCH_CHECK();
  }
  k_lov_finalize<<<1, 256, 0, s>>>((const double*)(sc + l.part), gts, K, nt, (float*)(sc + l.fin), loss);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_lovasz_bwd(const float* seg, const int64_t* target, int32_t B, int32_t K, int32_t h, int32_t w,
                              int32_t Himg, int32_t Wimg, int32_t ignore_index, void* scratch, const float* grad_loss,
                              float* dseg, void* stream) {
  LovArgs a;
  const int st = lov_make(seg, target, B, K, h, w, Himg, Wimg, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && dseg);
  cudaStream_t s = (cudaStream_t)stream;
  const LovLayout l = lov_layout(a);
  const char* sc = (const char*)scratch;
  return up_bwd_launch<k_lov_bwd_tile>(a, s, dseg, (const float2*)(sc + l.ms), (const float*)(sc + l.ge),
                                       (const float*)(sc + l.fin), grad_loss);
}

// ==================================================================================================================
// Fused OHEM cross-entropy of the contrast wrappers (FSOhemCELoss, and the seg term of FSAuxOhemCELoss,
// lib/loss/loss_helper.py:215-281): replaces
//   F.interpolate(seg, (Himg,Wimg), bilinear, align_corners=True) + softmax + gather of the target probability + sort of
//   the labelled pixels' p_t + nn.CrossEntropyLoss(weight, reduction='none') + the selection p_t < threshold
// and its autograd backward, without materialising the (B,K,Himg,Wimg) logits or probabilities and without a host sync.
// m = min(min_kept, n - 1) over the n counted pixels; threshold = max(kth, fp32(thresh)), kth the m-th smallest p_t
// (0-based); the loss sums w_t * nll over the pixels with p_t < threshold (strict: a tie at the threshold is all out).
//   k_segce_fwd<true>  the seg CE tile pass: per label pixel lse (kept for the backward), p_t and w_t * nll; integer
//                      counts of n and of p_t < thresh
//   k_ohem_decide      count(p_t < thresh) > m means kth < thresh: threshold = fp32(thresh), exact, and the select levels
//                      below exit at once (the usual training case); n = 0 takes the same exit
//   k_ohem_hist/scan   otherwise an exact radix select of the m-th smallest key over three levels of 11/11/10 bits of
//                      the p_t bits (p_t >= 0: the raw fp32 bits sort in value order); per level an integer histogram of
//                      the pixels matching the prefix so far, and a one-CTA scan that picks the digit holding rank m.
//                      State on the device, integer atomics only: the result does not depend on scheduling.
//   k_ohem_sum         per-CTA sums of w_t * nll (fp64) and counts over p_t < threshold, fixed tiles of OHEM_TILE pixels
//   k_ohem_finalize    fixed-order fp64 sum of the partials: sum / count ('mean', NaN for an empty selection, as the
//                      reference's mean of nothing) or the sum; 0 when no pixel counts.  Bit-reproducible.
//   k_segce_bwd_tile<true>  the seg CE backward with coefficient grad * w_t / count ('mean') or grad * w_t ('sum') at
//                      the pixels whose stored p_t < threshold, 0 elsewhere (dseg to the last ulp or two, fp32 atomics)
// First-order HBM bytes at B=8, K=19, 128x256 -> 512x1024 (N = 4.19 M): the tile pass reads seg (19.9 MB) and the labels
// (33.6 MB) and writes lse, p_t and w_t * nll (50.3 MB); each select level re-reads p_t (16.8 MB); the sum reads p_t and
// w_t * nll (33.6 MB); the backward reads the labels, lse, p_t and seg and writes dseg (DESIGN §4).
namespace pcl {

constexpr int OHEM_BINS = 2048;                      // 11-bit digits (the last level uses 10 of them)
constexpr int OHEM_THREADS = 256;
constexpr int OHEM_ITEMS = 8;
constexpr int OHEM_TILE = OHEM_THREADS * OHEM_ITEMS;  // pixels per k_ohem_sum CTA
constexpr int OHEM_HIST_CTAS = 1024;

// At byte 0 of the scratch (layout documented in pcl.h): the first four words are the finished forward's result.
struct OhemState {
  float loss, denom, threshold;   // loss; the backward's denominator (selected count for 'mean', 1 for 'sum'); threshold
  int select;                     // 1 when the select levels ran (count(p_t < thresh) <= m)
  int n, below, count, rank;      // counted pixels; p_t < thresh; selected pixels; rank still to find in the select
  uint32_t prefix;                // key bits found so far
};
static_assert(sizeof(OhemState) <= 256, "p_t starts at byte 256 of the scratch (pcl.h)");

__global__ void __launch_bounds__(32)
k_ohem_decide(OhemState* __restrict__ st, int64_t min_kept, float thresh) {
  if (threadIdx.x != 0) return;
  const int64_t n = st->n;
  const int64_t m = min(min_kept, n - 1);
  const bool sel = n > 0 && (int64_t)st->below <= m;
  st->select = sel ? 1 : 0;
  st->rank = sel ? (int)m : 0;
  st->prefix = 0u;
  st->threshold = thresh;                          // the select overwrites it with max(kth, thresh)
}

// level 0: bits 31..21 of every counted key; level 1: bits 20..10 of the keys whose bits 31..21 equal the prefix;
// level 2: bits 9..0 of the keys whose bits 31..10 equal the prefix
__global__ void __launch_bounds__(OHEM_THREADS)
k_ohem_hist(const float* __restrict__ p, int64_t N, int level, const OhemState* __restrict__ st, int* __restrict__ hist) {
  __shared__ int s_h[OHEM_BINS];
  if (!st->select) return;                         // uniform over the grid: the threshold decided
  const uint32_t prefix = st->prefix;
  const int shift = level == 0 ? 21 : (level == 1 ? 10 : 0);
  const int hi = level == 1 ? 21 : 10;
  const uint32_t mask = level == 2 ? 1023u : 2047u;
  for (int i = threadIdx.x; i < OHEM_BINS; i += OHEM_THREADS) s_h[i] = 0;
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * OHEM_THREADS + threadIdx.x; i < N; i += (int64_t)gridDim.x * OHEM_THREADS) {
    const float v = p[i];
    if (v != v) continue;                          // NaN: the pixel does not count
    const uint32_t key = __float_as_uint(v);
    if (level == 0 || (key >> hi) == prefix) atomicAdd(&s_h[(key >> shift) & mask], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < OHEM_BINS; i += OHEM_THREADS)
    if (s_h[i]) atomicAdd(&hist[level * OHEM_BINS + i], s_h[i]);
}

// One CTA: exclusive scan of the level's 2048 counts (two per thread); the thread whose bins hold rank r appends the
// digit to the prefix and keeps the rank within it.  After level 2 the prefix is the key of the m-th smallest p_t.
__global__ void __launch_bounds__(1024)
k_ohem_scan(int level, float thresh, OhemState* __restrict__ st, const int* __restrict__ hist) {
  __shared__ int s_w[32];
  if (!st->select) return;
  const int a0 = hist[level * OHEM_BINS + 2 * threadIdx.x], a1 = hist[level * OHEM_BINS + 2 * threadIdx.x + 1];
  const int s = a0 + a1;
  const int excl = block_exclusive_scan_1024(s, s_w);
  const int r = st->rank;
  int d = -1, nr = 0;
  if (r >= excl && r < excl + a0) { d = 2 * threadIdx.x; nr = r - excl; }
  else if (r >= excl + a0 && r < excl + s) { d = 2 * threadIdx.x + 1; nr = r - excl - a0; }
  __syncthreads();                                 // every thread has read the rank
  if (d >= 0) {
    const uint32_t prefix = (st->prefix << (level == 2 ? 10 : 11)) | (uint32_t)d;
    st->prefix = prefix;
    st->rank = nr;
    if (level == 2) st->threshold = fmaxf(__uint_as_float(prefix), thresh);
  }
}

__global__ void __launch_bounds__(OHEM_THREADS)
k_ohem_sum(const float* __restrict__ p, const float* __restrict__ wnll, int64_t N, const OhemState* __restrict__ st,
           double* __restrict__ part_s, int* __restrict__ part_c) {
  __shared__ double s_d[OHEM_THREADS / 32];
  __shared__ int s_c[OHEM_THREADS / 32];
  const float thr = st->threshold;
  const int64_t base = (int64_t)blockIdx.x * OHEM_TILE;
  double acc = 0.0;
  int c = 0;
  for (int r = 0; r < OHEM_ITEMS; ++r) {
    const int64_t i = base + r * OHEM_THREADS + threadIdx.x;
    if (i < N && p[i] < thr) { acc += (double)wnll[i]; ++c; }     // NaN (not counted) compares false
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  c = warp_sum_i(c);
  if ((threadIdx.x & 31) == 0) { s_d[threadIdx.x >> 5] = acc; s_c[threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sd = 0.0;
    int sc = 0;
    for (int w = 0; w < OHEM_THREADS / 32; ++w) { sd += s_d[w]; sc += s_c[w]; }    // fixed order
    part_s[blockIdx.x] = sd;
    part_c[blockIdx.x] = sc;
  }
}

__global__ void __launch_bounds__(1024)
k_ohem_finalize(const double* __restrict__ part_s, const int* __restrict__ part_c, int64_t nt, int reduction,
                OhemState* __restrict__ st, float* __restrict__ out) {
  block_sum2_1024<double, int64_t>(part_s, part_c, nt, [&](const double& sum, const int64_t& cnt) {
    float loss;
    if (st->n == 0) loss = 0.f;                                   // no labelled pixel: 0, zero gradient
    else if (reduction == 0) loss = (float)(sum / (double)cnt);   // 0 / 0 = NaN: the mean of an empty selection
    else loss = (float)sum;
    st->loss = loss;
    st->denom = reduction == 0 ? (float)cnt : 1.f;
    st->count = (int)cnt;
    out[0] = loss;
  });
}

}  // namespace pcl

namespace {

struct OhemLayout {
  size_t p, lse, wnll, hist, part_s, part_c, total;
  int64_t ntiles;
};

// state (byte 0) | p_t (byte 256, as pcl.h documents) | lse | w_t * nll | 3 histograms | partial sums, counts
OhemLayout ohem_layout(int64_t N) {
  OhemLayout l;
  l.ntiles = ceil_div64(N, OHEM_TILE);
  size_t o = align256(sizeof(OhemState));
  l.p = o;      o = align256(o + (size_t)N * 4);
  l.lse = o;    o = align256(o + (size_t)N * 4);
  l.wnll = o;   o = align256(o + (size_t)N * 4);
  l.hist = o;   o = align256(o + (size_t)3 * OHEM_BINS * 4);
  l.part_s = o; o = align256(o + (size_t)l.ntiles * 8);
  l.part_c = o; o = align256(o + (size_t)l.ntiles * 4);
  l.total = o;
  return l;
}

int ohem_make(const float* seg, const int64_t* target, const float* weight, int B, int K, int h, int w, int H, int W,
              int ignore_index, SegCeArgs* a) {
  if (!seg || !target) return PCL_ERR_ARG;
  const int st = sort_geometry(B, K, h, w, H, W, a);
  if (st != PCL_OK) return st;
  return make_ce(seg, target, weight, B, K, h, w, H, W, ignore_index, a);
}

}  // namespace

extern "C" int64_t pcl_ohem_ce_scratch_bytes(int32_t B, int32_t K, int32_t h, int32_t w, int32_t Himg, int32_t Wimg) {
  UpGeom g;
  const int st = sort_geometry(B, K, h, w, Himg, Wimg, &g);
  if (st != PCL_OK) return st;
  return (int64_t)ohem_layout((int64_t)B * Himg * Wimg).total;
}

extern "C" int pcl_ohem_ce_fwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K,
                               int32_t h, int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index, float thresh,
                               int64_t min_kept, int32_t reduction, void* scratch, float* loss, void* stream) {
  SegCeArgs a;
  int st = ohem_make(seg, target, class_weight, B, K, h, w, Himg, Wimg, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && loss && min_kept >= 1 && (reduction == 0 || reduction == 1));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t N = (int64_t)B * Himg * Wimg;
  const OhemLayout l = ohem_layout(N);
  char* sc = (char*)scratch;
  OhemState* state = (OhemState*)sc;
  float* p = (float*)(sc + l.p);
  float* wnll = (float*)(sc + l.wnll);
  int* hist = (int*)(sc + l.hist);
  PCL_CUDA(cudaMemsetAsync(state, 0, sizeof(OhemState), s));
  PCL_CUDA(cudaMemsetAsync(hist, 0, (size_t)3 * OHEM_BINS * sizeof(int), s));
  st = segce_fwd_launch<true>(a, (float*)(sc + l.lse), nullptr, nullptr, OhemPix{p, wnll, &state->n, thresh}, s);
  if (st != PCL_OK) return st;
  k_ohem_decide<<<1, 32, 0, s>>>(state, min_kept, thresh);
  PCL_LAUNCH_CHECK();
  const int64_t tiles = ceil_div64(N, OHEM_TILE);
  const unsigned hist_ctas = (unsigned)(tiles < OHEM_HIST_CTAS ? tiles : OHEM_HIST_CTAS);
  for (int level = 0; level < 3; ++level) {
    k_ohem_hist<<<hist_ctas, OHEM_THREADS, 0, s>>>(p, N, level, state, hist);
    PCL_LAUNCH_CHECK();
    k_ohem_scan<<<1, 1024, 0, s>>>(level, thresh, state, hist);
    PCL_LAUNCH_CHECK();
  }
  k_ohem_sum<<<(unsigned)l.ntiles, OHEM_THREADS, 0, s>>>(p, wnll, N, state, (double*)(sc + l.part_s),
                                                         (int*)(sc + l.part_c));
  PCL_LAUNCH_CHECK();
  k_ohem_finalize<<<1, 1024, 0, s>>>((const double*)(sc + l.part_s), (const int*)(sc + l.part_c), l.ntiles, reduction,
                                     state, loss);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_ohem_ce_bwd(const float* seg, const int64_t* target, const float* class_weight, int32_t B, int32_t K,
                               int32_t h, int32_t w, int32_t Himg, int32_t Wimg, int32_t ignore_index,
                               const void* scratch, const float* grad_loss, float* dseg, void* stream) {
  SegCeArgs a;
  const int st = ohem_make(seg, target, class_weight, B, K, h, w, Himg, Wimg, ignore_index, &a);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(scratch && dseg);
  const OhemLayout l = ohem_layout((int64_t)B * Himg * Wimg);
  const char* sc = (const char*)scratch;
  return up_bwd_launch<k_segce_bwd_tile<true>>(a, (cudaStream_t)stream, dseg, (const float*)(sc + l.lse),
                                                (const float*)sc, grad_loss, (const float*)(sc + l.p));
}
