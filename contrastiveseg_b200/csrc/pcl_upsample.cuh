// Tile geometry of the fused bilinear up-sampling kernels (F.interpolate(..., mode='bilinear', align_corners=True)),
// shared by the seg CE, the RMI, the Lovasz-softmax and the OHEM CE losses (all in pcl_segce.cu).  A CTA owns a BT x BTY
// tile of label pixels of one image; the source logits the tile reads form a ys_n x xs_n patch starting at
// (ys_base, xs_base), staged per class chunk (up_stage).  The backward maps a per-pixel gradient G[class][row][col] of the
// tile through the transposed bilinear map into dseg (up_tile_flush).
#pragma once
#include "pcl_common.cuh"

namespace pcl {

constexpr int BT = 32;                 // tile width  (label pixels)
constexpr int BTY = 8;                 // tile height: 32 x 8 = 256 threads per CTA -> several CTAs per SM hide the
                                       // load latency of the bulk-synchronous phases (a 32 x 32 tile ran 1 CTA/SM)
constexpr int SRC_MAX = 34;            // source cells per tile edge (scale >= 1: up to 32 + 2)
constexpr int KC_FWD_MAX = 32;         // classes staged per forward pass (one pass for K <= 32: one exposed load latency)
constexpr int KC_BWD_MAX = 24;         // classes per backward pass (one pass for K <= 24: fewer bulk-synchronous phases)

// Logits (B, K, h, w) up-sampled to the label grid (B, H, W).
struct UpGeom {
  int B, K, h, w, H, W;
  float ry, rx;                 // (h-1)/(H-1), (w-1)/(W-1)   (align_corners=True)
};

// PCL_ERR_ARG on a non-positive dimension; otherwise fills g.
static inline int up_geometry(int B, int K, int h, int w, int H, int W, UpGeom* g) {
  if (B <= 0 || K <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) return PCL_ERR_ARG;
  g->B = B; g->K = K; g->h = h; g->w = w; g->H = H; g->W = W;
  g->ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
  g->rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  return PCL_OK;
}

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

__device__ __forceinline__ void src_coord(int o, float r, int in_size, int& i0, int& i1, float& l1) {
  const float s = r * (float)o;                       // ATen area_pixel_compute_source_index, align_corners=True
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

// Source patch geometry of a tile (identical for every thread of the CTA).
struct UpTile {
  int X0, Y0, nx, ny;                  // first label column / row, valid columns / rows of the tile
  int ys_base, xs_base, ys_n, xs_n;    // source patch
};

// Source rows / columns (and bilinear weights) of the tile's label rows / columns into shared memory; then the patch.
// Every thread of the CTA calls it (it contains a barrier).
__device__ __forceinline__ UpTile up_tile_coords(int X0, int Y0, int H, int W, int h, int w, float ry, float rx,
                                                 int* s_y0, int* s_y1, float* s_ly, int* s_x0, int* s_x1, float* s_lx) {
  if (threadIdx.x < BT) {
    int i0, i1; float l;
    if (threadIdx.x < BTY) {
      src_coord(min(Y0 + (int)threadIdx.x, H - 1), ry, h, i0, i1, l);
      s_y0[threadIdx.x] = i0; s_y1[threadIdx.x] = i1; s_ly[threadIdx.x] = l;
    }
    src_coord(min(X0 + (int)threadIdx.x, W - 1), rx, w, i0, i1, l);
    s_x0[threadIdx.x] = i0; s_x1[threadIdx.x] = i1; s_lx[threadIdx.x] = l;
  }
  __syncthreads();
  UpTile g;
  g.X0 = X0; g.Y0 = Y0;
  g.ny = min(Y0 + BTY, H) - Y0; g.nx = min(X0 + BT, W) - X0;
  g.ys_base = s_y0[0]; g.xs_base = s_x0[0];
  g.ys_n = s_y1[g.ny - 1] - g.ys_base + 1; g.xs_n = s_x1[g.nx - 1] - g.xs_base + 1;
  return g;
}

// Bilinear weights and patch offsets of this thread's label pixel (column tx, row ty of the tile) in the staged patch
struct UpPix {
  float w00, w01, w10, w11;
  int i00, i01, i10, i11;
  float ly, lx;                        // the row / column weights the four above are built from
};

__device__ __forceinline__ UpPix up_pix(const UpTile& g, int tx, int ty, const int* s_y0, const int* s_y1,
                                        const float* s_ly, const int* s_x0, const int* s_x1, const float* s_lx) {
  UpPix p;
  const int ly0 = s_y0[ty] - g.ys_base, ly1 = s_y1[ty] - g.ys_base, lx0 = s_x0[tx] - g.xs_base, lx1 = s_x1[tx] - g.xs_base;
  const float ly = s_ly[ty], lx = s_lx[tx];
  p.ly = ly; p.lx = lx;
  p.w00 = (1.f - ly) * (1.f - lx); p.w01 = (1.f - ly) * lx; p.w10 = ly * (1.f - lx); p.w11 = ly * lx;
  p.i00 = ly0 * g.xs_n + lx0; p.i01 = ly0 * g.xs_n + lx1; p.i10 = ly1 * g.xs_n + lx0; p.i11 = ly1 * g.xs_n + lx1;
  return p;
}

// The up-sampled logit of the pixel from one staged class plane s
__device__ __forceinline__ float up_logit(const UpPix& p, const float* s) {
  return p.w00 * s[p.i00] + p.w01 * s[p.i01] + p.w10 * s[p.i10] + p.w11 * s[p.i11];
}

// Copies the ys_n x xs_n source patch at (ys_base, xs_base) of classes [c0, c0 + cn) of image b into S[cc][pitch], by
// every thread of the 256-thread CTA.  The caller syncs before reading S.
__device__ __forceinline__ void up_stage(const UpGeom& a, const float* seg, int b, int c0, int cn, int ys_base,
                                         int xs_base, int ys_n, int xs_n, int pitch, float* S) {
  const int patch = ys_n * xs_n;
  const int64_t hw = (int64_t)a.h * a.w;
  for (int i = threadIdx.x; i < cn * patch; i += BT * BTY) {
    const int cc = i / patch, r = i - cc * patch;
    const int yy = r / xs_n, xx = r - yy * xs_n;
    S[cc * pitch + r] = seg[((int64_t)b * a.K + c0 + cc) * hw + (int64_t)(ys_base + yy) * a.w + xs_base + xx];
  }
}

// The transposed bilinear map of the tile, once per CTA (it is the same for every class and row): weight of label
// column k in source column xs (s_wx), of label row k in source row ys (s_wy), and the label range [klo, khi] inside
// a source cell's footprint.  Row stride BT + 1 / BTY + 1: different source cells of one k fall into different banks.
// s_wx: SRC_MAX * (BT + 1) floats, s_wy: SRC_MAX * (BTY + 1), s_xlo / s_xhi / s_ylo / s_yhi: SRC_MAX.  Caller syncs.
__device__ __forceinline__ void up_tile_tables(const UpTile& g, float ry, float rx, const int* s_y0, const int* s_y1,
                                               const float* s_ly, const int* s_x0, const int* s_x1, const float* s_lx,
                                               float* s_wx, float* s_wy, short* s_xlo, short* s_xhi, short* s_ylo,
                                               short* s_yhi) {
  const float inv_rx = rx > 0.f ? 1.f / rx : 0.f, inv_ry = ry > 0.f ? 1.f / ry : 0.f;
  for (int i = threadIdx.x; i < g.xs_n * BT; i += BT * BTY) {
    const int xs = i / BT, k = i - xs * BT, xg = g.xs_base + xs;
    float wgt = 0.f;
    if (k < g.nx) {
      if (s_x0[k] == xg) wgt += 1.f - s_lx[k];
      if (s_x1[k] == xg) wgt += s_lx[k];
    }
    s_wx[xs * (BT + 1) + k] = wgt;
  }
  for (int i = threadIdx.x; i < g.ys_n * BTY; i += BT * BTY) {
    const int ysl = i / BTY, k = i - ysl * BTY, yg = g.ys_base + ysl;
    float wgt = 0.f;
    if (k < g.ny) {
      if (s_y0[k] == yg) wgt += 1.f - s_ly[k];
      if (s_y1[k] == yg) wgt += s_ly[k];
    }
    s_wy[ysl * (BTY + 1) + k] = wgt;
  }
  if (threadIdx.x < g.xs_n) {
    const int xg = g.xs_base + threadIdx.x;
    int klo = 0, khi = g.nx - 1;
    if (rx > 0.f) {
      klo = max(0, (int)floorf(((float)xg - 1.f) * inv_rx) - 1 - g.X0);
      khi = min(g.nx - 1, (int)ceilf(((float)xg + 1.f) * inv_rx) + 1 - g.X0);
    }
    s_xlo[threadIdx.x] = (short)klo; s_xhi[threadIdx.x] = (short)khi;
  }
  if (threadIdx.x >= 64 && threadIdx.x < 64 + g.ys_n) {
    const int ysl = threadIdx.x - 64, yg = g.ys_base + ysl;
    int klo = 0, khi = g.ny - 1;
    if (ry > 0.f) {
      klo = max(0, (int)floorf(((float)yg - 1.f) * inv_ry) - 1 - g.Y0);
      khi = min(g.ny - 1, (int)ceilf(((float)yg + 1.f) * inv_ry) + 1 - g.Y0);
    }
    s_ylo[ysl] = (short)klo; s_yhi[ysl] = (short)khi;
  }
}

// G [cn][BTY][BT] (gradient w.r.t. the virtual up-sampled logits of the tile, written and synced by the caller) ->
//   B  x direction:  Hx[c][row][xs] = sum_x wx(x, xs) * G[c][row][x]   (only the label columns whose footprint
//                    touches source column xs)
//   C  y direction + flush: dseg_c0[c * hw + ys * w + xs] += sum_row wy(row, ys) * Hx[c][row][xs]  (global atomics
//                    only on the source cells of the tile; a cell is shared by at most 4 tiles)
// Hx: cn * BTY * SRC_MAX floats.  dseg_c0 points at the first class plane of the chunk.  Caller syncs afterwards.
__device__ __forceinline__ void up_tile_flush(const UpTile& g, int cn, const float* G, float* Hx, const float* s_wx,
                                              const float* s_wy, const short* s_xlo, const short* s_xhi,
                                              const short* s_ylo, const short* s_yhi, float* dseg_c0, int64_t hw,
                                              int w) {
  for (int i = threadIdx.x; i < cn * BTY * g.xs_n; i += BT * BTY) {
    const int xs = i % g.xs_n, row = (i / g.xs_n) % BTY, cc = i / (g.xs_n * BTY);
    const int klo = s_xlo[xs], khi = s_xhi[xs];
    const float* gr = G + ((size_t)cc * BTY + row) * BT;
    const float* wr = s_wx + xs * (BT + 1);
    float acc = 0.f;
    for (int k = klo; k <= khi; ++k) acc += wr[k] * gr[k];
    Hx[((size_t)cc * BTY + row) * SRC_MAX + xs] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cn * g.ys_n * g.xs_n; i += BT * BTY) {
    const int xs = i % g.xs_n, ysl = (i / g.xs_n) % g.ys_n, cc = i / (g.xs_n * g.ys_n);
    const int yg = g.ys_base + ysl;
    const int klo = s_ylo[ysl], khi = s_yhi[ysl];
    const float* wr = s_wy + ysl * (BTY + 1);
    float acc = 0.f;
    for (int k = klo; k <= khi; ++k) acc += wr[k] * Hx[((size_t)cc * BTY + k) * SRC_MAX + xs];
    if (acc != 0.f) atomicAdd(&dseg_c0[(int64_t)cc * hw + (int64_t)yg * w + g.xs_base + xs], acc);
  }
}

// Upper bound of the source cells a rows x cols block of label pixels touches (ys_n * xs_n), + 1 to de-phase the class
// planes.
static inline int up_patch_pitch(const UpGeom& a, int rows, int cols) {
  const int py = (int)((float)(rows - 1) * a.ry) + 3, px = (int)((float)(cols - 1) * a.rx) + 3;
  return (py < a.h + 1 ? py : a.h + 1) * (px < a.w + 1 ? px : a.w + 1) + 1;
}

// Forward launch plan: kc classes staged per pass (at most KC_FWD_MAX), fewer while the kc source patches of `pitch`
// floats and `extra` bytes exceed 96 KB (two CTAs per SM).
struct UpPlan {
  int pitch, kc;
  size_t smem;
};

static inline int up_fwd_plan(const UpGeom& a, int pitch, size_t extra, UpPlan* p) {
  int kc = a.K < KC_FWD_MAX ? a.K : KC_FWD_MAX;
  while (kc > 1 && extra + (size_t)kc * pitch * sizeof(float) > 96 * 1024) --kc;
  p->pitch = pitch; p->kc = kc;
  p->smem = extra + (size_t)kc * pitch * sizeof(float);
  return p->smem > 200 * 1024 ? PCL_ERR_UNSUPPORTED : PCL_OK;
}

}  // namespace pcl
