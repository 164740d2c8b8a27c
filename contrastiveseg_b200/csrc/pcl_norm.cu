// Projection head kernels.
// (1) L2 normalise over the channel dim of an NCHW tensor (SURVEY §8 row a1).
// Replaces lib/models/modules/projection.py:24  F.normalize(x, p=2, dim=1)  and its autograd backward.
// HBM-bound: forward reads x once and writes y once (2 * B*D*HW*4 bytes); backward reads x and gy once and
// writes gx once.  One CTA covers 32 consecutive pixels x all D channels: lanes run along the pixel
// dimension (coalesced 128 B rows), the 8 warps split the channels and keep their values in registers.
#include "pcl_common.cuh"
#include "ptx_sm90.cuh"

namespace pcl {

constexpr int NW = 8;            // warps per CTA (channel groups)
constexpr int VMAX = 32;         // register-resident channels per thread (D <= NW * VMAX = 256)

template <bool BWD>
__global__ void __launch_bounds__(NW * 32)
k_l2norm(const float* __restrict__ x, const float* __restrict__ gy, float* __restrict__ out, int D, int64_t HW,
         int64_t tiles_per_image) {
  __shared__ float s_ss[NW][32];
  __shared__ float s_dot[NW][32];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int64_t b = blockIdx.x / tiles_per_image;
  const int64_t p = (blockIdx.x - b * tiles_per_image) * 32 + lane;
  const bool ok = p < HW;
  const int64_t base = b * (int64_t)D * HW + p;
  float xv[VMAX], gv[VMAX];
  float ss = 0.f, dot = 0.f;
#pragma unroll
  for (int i = 0; i < VMAX; ++i) {
    const int d = g + i * NW;
    xv[i] = 0.f; gv[i] = 0.f;
    if (ok && d < D) {
      xv[i] = x[base + (int64_t)d * HW];
      if (BWD) gv[i] = gy[base + (int64_t)d * HW];
    }
    ss = fmaf(xv[i], xv[i], ss);
    if (BWD) dot = fmaf(xv[i], gv[i], dot);
  }
  // channels beyond NW*VMAX (D > 256): streamed, re-read in the second pass
  for (int d = g + VMAX * NW; d < D; d += NW) {
    if (ok) {
      float v = x[base + (int64_t)d * HW];
      ss = fmaf(v, v, ss);
      if (BWD) dot = fmaf(v, gy[base + (int64_t)d * HW], dot);
    }
  }
  s_ss[g][lane] = ss;
  if (BWD) s_dot[g][lane] = dot;
  __syncthreads();
  float tss = 0.f, tdot = 0.f;
#pragma unroll
  for (int k = 0; k < NW; ++k) { tss += s_ss[k][lane]; if (BWD) tdot += s_dot[k][lane]; }
  const float nrm = sqrtf(tss);
  const bool clamped = nrm < 1e-12f;
  const float inv = 1.f / fmaxf(nrm, 1e-12f);
  // d/dx [x / max(|x|, eps)]:  g/|x| - x (x.g)/|x|^3   (denominator constant when clamped)
  const float coef = (BWD && !clamped) ? tdot * inv * inv * inv : 0.f;
  if (!ok) return;
#pragma unroll
  for (int i = 0; i < VMAX; ++i) {
    const int d = g + i * NW;
    if (d < D) out[base + (int64_t)d * HW] = BWD ? (gv[i] * inv - xv[i] * coef) : xv[i] * inv;
  }
  for (int d = g + VMAX * NW; d < D; d += NW) {
    float v = x[base + (int64_t)d * HW];
    out[base + (int64_t)d * HW] = BWD ? (gy[base + (int64_t)d * HW] * inv - v * coef) : v * inv;
  }
}

}  // namespace pcl

using namespace pcl;

static int launch_norm(bool bwd, const float* x, const float* gy, float* out, int32_t B, int32_t D, int64_t HW,
                       void* stream) {
  PCL_REQUIRE(x && out && B > 0 && D > 0 && HW > 0);
  if (bwd) PCL_REQUIRE(gy);
  const int64_t tiles = ceil_div64(HW, 32);
  const int64_t blocks = tiles * B;
  PCL_REQUIRE(blocks < (1ll << 31));
  cudaStream_t s = (cudaStream_t)stream;
  if (bwd) k_l2norm<true><<<(unsigned)blocks, NW * 32, 0, s>>>(x, gy, out, D, HW, tiles);
  else     k_l2norm<false><<<(unsigned)blocks, NW * 32, 0, s>>>(x, nullptr, out, D, HW, tiles);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_l2norm_fwd(const float* x, float* y, int32_t B, int32_t D, int64_t HW, void* stream) {
  return launch_norm(false, x, nullptr, y, B, D, HW, stream);
}

extern "C" int pcl_l2norm_bwd(const float* x, const float* gy, float* gx, int32_t B, int32_t D, int64_t HW,
                              void* stream) {
  return launch_norm(true, x, gy, gx, B, D, HW, stream);
}

// (2) The head's last 1x1 convolution + L2 normalise as wgmma GEMMs, forward and backward (SURVEY §8f row 2).
// Replaces lib/models/modules/projection.py:17-24  F.normalize(Conv2d(Cin -> 256, k=1)(x), p=2, dim=1)  and its
// autograd backward.  bf16 operands, fp32 accumulate (the precision="bf16" contract of the tensor sweep).
//
//   k_proj_pack    W (256, Cin) fp32 -> Wk (256, Cin up to 64) bf16 and Wt (Cin up to 256, 256) bf16, zero-padded
//   k_proj_fwd     CTA = 128 pixels of one image x 256 channels; A = x tile converted fp32 NCHW -> bf16 by the threads
//                  into the K-major 128B-swizzled layout (register-staged one K-block ahead), B = Wk by TMA (3 stages).
//                  Epilogue on the fragment: + bias, row norm = thread-local sum + two quad shuffles, zn and inv_norm.
//   k_proj_dgrad   prologue: gz = (gzn - zn <zn, gzn>) inv (clamped: gzn inv), bf16, into shared memory (the A operand)
//                  and into the caller's gz workspace (B, 256, HW up to 64, zero tail); then gx^T = gz . Wt^T in
//                  256-channel passes, the next pass's Wt loaded by TMA during the current pass's gx stores.
//   k_proj_wgrad   split-K over pixels: gW partial (256 x Cin+1) = gz . x^T; A = gz by TMA, B = x tile converted by
//                  the threads into the MN-major layout.  Channel Cin of the converted tile is 1 (valid pixels), so
//                  column Cin of the product is gb = sum_p gz[:, p].
//   k_proj_reduce  fixed-order sum of the split partials -> gW, gb (bit-reproducible).
// Pixel tiles never straddle images, so any H x W works; the activations are read with scalar loads (per-image rows of
// HW elements are not 16-byte aligned in general), coalesced along the pixel dimension.
// Activation element type T (x, zn, gzn, gx) is float or __nv_bfloat16.  bf16 x goes into the bf16 operand tile as its
// raw bits (what the fp32 path's round-to-bf16 gives for the same values), zn and gzn convert to fp32 on load (exact),
// and every sum runs in fp32 in the same order for both, so a bf16 call computes what the fp32 call computes on the
// converted inputs; bf16 zn and gx are the fp32 values rounded once to nearest-even.  inv_norm, the bf16 gz workspace,
// the split-K partials, gW and gb are fp32 / bf16 alike for both types.

namespace pcl {
namespace proj {

constexpr int DOUT = 256;                        // output channels (proj_dim)
constexpr int BM = 128;                          // pixels per forward / dgrad tile
constexpr int BK = 64;                           // K-block (128 bytes of bf16 per row)
constexpr int WB = 64;                           // pixels per wgrad K-block
constexpr int NT = 256;                          // two consumer warpgroups, no producer warpgroup
constexpr int WG_ROWS_BYTES = 64 * 128;          // warpgroup 1's 64 rows inside a [128 x 64] bf16 K-block
constexpr int A_KB = BM * BK * 2;                // 16 KB
constexpr int W_KB = DOUT * BK * 2;              // 32 KB
constexpr int FWD_WSTAGES = 3;
constexpr float NORM_EPS_INV = 1e12f;            // 1 / F.normalize's eps

struct FwdSmem {
  uint8_t w[FWD_WSTAGES][W_KB];
  uint8_t a[2][A_KB];
  uint64_t full[FWD_WSTAGES];
  float bias[DOUT];
};
struct DgradSmem {
  uint8_t a[DOUT / BK][A_KB];                    // gz tile, 4 K-blocks of 64 channels
  uint8_t wt[DOUT / BK][W_KB];                   // one 256-channel pass of Wt
  uint64_t full;
  float red[8][32];
};
struct WgradSmem {
  uint8_t a[3][A_KB];                            // gz rows n0 .. n0 + 127 x 64 pixels (TMA)
  uint8_t b[2][W_KB];                            // x: 64 pixels x 4 chunks of 64 channels, MN-major
  uint64_t full[3];
};
static_assert(sizeof(FwdSmem) + 1024 <= 227 * 1024, "shared memory of one H100 block");
static_assert(sizeof(DgradSmem) + 1024 <= 227 * 1024, "shared memory of one H100 block");
static_assert(sizeof(WgradSmem) + 1024 <= 227 * 1024, "shared memory of one H100 block");

template <class T>
__device__ __forceinline__ T& aligned_smem(uint8_t* raw) {
  return *reinterpret_cast<T*>(raw + ((1024u - (ptx::smem_u32(raw) & 1023u)) & 1023u));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// mbarrier wait without ptx::mbar_wait's timeout printf: a call in the kernel serialises every wgmma
__device__ __forceinline__ void wait_full(uint64_t* bar, uint32_t parity) {
  for (uint32_t spins = 0; !ptx::mbar_try_wait(bar, parity);)
    if (++spins > (1u << 24)) __trap();
}

// 1 / max(|z|, 1e-12) from |z|^2.  Clamped rows (the reciprocal would reach 1e12) get exactly 1e12, which is also how
// the backward recognises them.
__device__ __forceinline__ float inv_norm_of(float ss) {
#ifdef PCL_EMULATION
  const float r = 1.f / sqrtf(ss);
#else
  const float r = rsqrtf(ss);        // MUFU.RSQ: no IEEE-division / sqrt slow-path call next to the wgmma
#endif
  return r < NORM_EPS_INV ? r : NORM_EPS_INV;
}

// One channel value of the activation tile between its load and its store into the swizzled bf16 tile: fp32 values are
// rounded to bf16 at the store; a bf16 activation already is the GEMM operand, so its raw 16 bits are carried through
// unconverted (bf16 -> fp32 -> bf16 would be the identity).  Keeping the raw bits also keeps every load of a K-block
// independent of any arithmetic until the tile store, so all of them are in flight together as in the fp32 path.
template <class T> struct Staged { using type = float; };
template <> struct Staged<__nv_bfloat16> { using type = uint16_t; };

// 8 channels [c, c + 8) of pixel p of one NCHW image -> v.  Channels >= Cin read as 0, channel `ones` as 1 (the wgrad's
// bias column); pixels >= HW read as 0.  Nothing beyond the tensor is dereferenced.
__device__ __forceinline__ void load8(const float* __restrict__ img, int Cin, int64_t HW, int c, int64_t p, int ones,
                                      float (&v)[8]) {
  const bool pv = p < HW;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int ch = c + i;
    v[i] = (pv && ch < Cin) ? img[(int64_t)ch * HW + p] : ((pv && ch == ones) ? 1.f : 0.f);
  }
}
__device__ __forceinline__ void load8(const __nv_bfloat16* __restrict__ img, int Cin, int64_t HW, int c, int64_t p,
                                      int ones, uint16_t (&v)[8]) {
  constexpr uint16_t BF16_ONE = 0x3F80;
  const uint16_t* __restrict__ bits = reinterpret_cast<const uint16_t*>(img);
  const bool pv = p < HW;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int ch = c + i;
    v[i] = (pv && ch < Cin) ? bits[(int64_t)ch * HW + p] : ((pv && ch == ones) ? BF16_ONE : (uint16_t)0);
  }
}
// 8 values -> one 16-byte chunk of a 128B-swizzled row (row `r` of a 1024-aligned tile, chunk index `ch` in [0, 8))
__device__ __forceinline__ void store8(uint8_t* tile, int r, int ch, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(tile + r * 128 + ((ch ^ (r & 7)) << 4)) = u;
}
__device__ __forceinline__ void store8(uint8_t* tile, int r, int ch, const uint16_t (&v)[8]) {
  uint4 u;
  u.x = v[0] | ((uint32_t)v[1] << 16); u.y = v[2] | ((uint32_t)v[3] << 16);
  u.z = v[4] | ((uint32_t)v[5] << 16); u.w = v[6] | ((uint32_t)v[7] << 16);
  *reinterpret_cast<uint4*>(tile + r * 128 + ((ch ^ (r & 7)) << 4)) = u;
}

// ------------------------------------------------------------------------------------------------------------------
__global__ void k_proj_pack(const float* __restrict__ w, int Cin, int cin64, int cin256, __nv_bfloat16* __restrict__ wk,
                            __nv_bfloat16* __restrict__ wt) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)DOUT * cin256) return;
  const int n = (int)(idx / cin256), c = (int)(idx % cin256);
  const __nv_bfloat16 v = __float2bfloat16(c < Cin ? w[(int64_t)n * Cin + c] : 0.f);
  if (c < cin64) wk[(int64_t)n * cin64 + c] = v;
  wt[(int64_t)c * DOUT + n] = v;
}

// ------------------------------------------------------------------------------------------------------------------
template <class T>
struct FwdArgs {
  const T* x; const float* bias; T* zn; float* inv_norm;
  int Cin, nkb; int64_t HW; int tiles_per_img;
};

template <class T>
__global__ void __launch_bounds__(NT, 1) k_proj_fwd(const __grid_constant__ CUtensorMap tmW, FwdArgs<T> a) {
  extern __shared__ uint8_t smem_raw[];
  FwdSmem& sm = aligned_smem<FwdSmem>(smem_raw);
  const int t = threadIdx.x, g = t >> 7, lane = t & 31, wt = t & 127;
  const int b = blockIdx.x / a.tiles_per_img;
  const int64_t p0 = (int64_t)(blockIdx.x - b * a.tiles_per_img) * BM;
  const T* img = a.x + (int64_t)b * a.Cin * a.HW;
  if (t == 0) {
    ptx::prefetch_tmap(&tmW);
    for (int s = 0; s < FWD_WSTAGES; ++s) ptx::mbar_init(&sm.full[s], 1);
    ptx::fence_barrier_init();
  }
  sm.bias[t] = a.bias ? a.bias[t] : 0.f;
  __syncthreads();
  if (t == 0)
    for (int kb = 0; kb < 2 && kb < a.nkb; ++kb) {
      ptx::mbar_arrive_expect_tx(&sm.full[kb], W_KB);
      ptx::tma_load_2d(sm.w[kb], &tmW, &sm.full[kb], kb * BK, 0);
    }
  // conversion items of this thread: pixel row wt, 16-byte channel chunks g, g + 2, g + 4, g + 6 of each K-block
  typename Staged<T>::type v[4][8];
#pragma unroll
  for (int j = 0; j < 4; ++j) load8(img, a.Cin, a.HW, 8 * (g + 2 * j), p0 + wt, -1, v[j]);
#pragma unroll
  for (int j = 0; j < 4; ++j) store8(sm.a[0], wt, g + 2 * j, v[j]);
  ptx::fence_proxy_async();

  float acc[128];
  const uint32_t a_off = g * WG_ROWS_BYTES;
  for (int kb = 0; kb < a.nkb; ++kb) {
    const int sa = kb & 1, sw = kb % FWD_WSTAGES;
    __syncthreads();                     // A[sa] complete; every wgmma of K-block kb - 1 retired (stage reuse below)
    if (t == 0 && kb + 2 < a.nkb) {
      const int s2 = (kb + 2) % FWD_WSTAGES;
      ptx::mbar_arrive_expect_tx(&sm.full[s2], W_KB);
      ptx::tma_load_2d(sm.w[s2], &tmW, &sm.full[s2], (kb + 2) * BK, 0);
    }
    const bool more = kb + 1 < a.nkb;
    if (more) {
#pragma unroll
      for (int j = 0; j < 4; ++j) load8(img, a.Cin, a.HW, (kb + 1) * BK + 8 * (g + 2 * j), p0 + wt, -1, v[j]);
    }
    wait_full(&sm.full[sw], (uint32_t)(kb / FWD_WSTAGES) & 1u);
    const uint32_t abase = ptx::smem_u32(sm.a[sa]) + a_off, wbase = ptx::smem_u32(sm.w[sw]);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      ptx::wgmma_m64n256k16<0>(acc, ptx::make_desc_kmajor_sw128(abase + k * 32), ptx::make_desc_kmajor_sw128(wbase + k * 32),
                               (kb | k) != 0 ? 1u : 0u);
    ptx::wgmma_commit();
    if (more) {
#pragma unroll
      for (int j = 0; j < 4; ++j) store8(sm.a[sa ^ 1], wt, g + 2 * j, v[j]);
      ptx::fence_proxy_async();
    }
    ptx::wgmma_wait<0>();
    ptx::fence_operands(acc);
  }

  // epilogue on the fragment: acc[4 i + 2 h + e] = pixel fr + 8 h of the warpgroup, channel 8 i + 2 q + e
  const int fr = 16 * (wt >> 5) + (lane >> 2), q = lane & 3;
  T* out = a.zn + (int64_t)b * DOUT * a.HW;
  // 2-byte zn: straight from the fragment a warp store would write 16-byte pieces of 4 channel rows; instead the tile
  // is staged [channel][pixel] in the retired weight stages and written out along pixels, 64 contiguous bytes per warp
  // store.  The row pitch of ZS_LD elements (68 words) spreads a fragment store's 4 channel pairs over distinct banks.
  constexpr int ZS_LD = BM + 8;
  static_assert(DOUT * ZS_LD * 2 <= sizeof(FwdSmem::w), "zn staging tile fits the weight stages");
  T* stage = reinterpret_cast<T*>(sm.w[0]);
  if constexpr (sizeof(T) == 2) __syncthreads();      // both warpgroups' last wgmma has read sm.w
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float z = acc[4 * i + 2 * h + e] + sm.bias[8 * i + 2 * q + e];
        acc[4 * i + 2 * h + e] = z;
        ss = fmaf(z, z, ss);
      }
    const float inv = inv_norm_of(quad_sum(ss));
    const int64_t p = p0 + g * 64 + fr + 8 * h;
    if (p < a.HW) {
      if (q == 0) a.inv_norm[(int64_t)b * a.HW + p] = inv;
      if constexpr (sizeof(T) == 4) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            out[(int64_t)(8 * i + 2 * q + e) * a.HW + p] = from_f32<T>(acc[4 * i + 2 * h + e] * inv);
      }
    }
    if constexpr (sizeof(T) == 2) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          stage[(8 * i + 2 * q + e) * ZS_LD + g * 64 + fr + 8 * h] = from_f32<T>(acc[4 * i + 2 * h + e] * inv);
    }
  }
  if constexpr (sizeof(T) == 2) {
    __syncthreads();
    for (int c = t >> 5; c < DOUT; c += NT / 32)
#pragma unroll
      for (int j = 0; j < BM / 32; ++j) {
        const int px = 32 * j + lane;
        if (p0 + px < a.HW) out[(int64_t)c * a.HW + p0 + px] = stage[c * ZS_LD + px];
      }
  }
}

// ------------------------------------------------------------------------------------------------------------------
template <class T>
struct DgradArgs {
  const T* zn; const T* gzn; const float* inv_norm; T* gx; __nv_bfloat16* gz;
  int Cin, npass; int64_t HW, HWp; int tiles_per_img;
};

template <class T>
__global__ void __launch_bounds__(NT, 1) k_proj_dgrad(const __grid_constant__ CUtensorMap tmWt, DgradArgs<T> a) {
  extern __shared__ uint8_t smem_raw[];
  DgradSmem& sm = aligned_smem<DgradSmem>(smem_raw);
  const int t = threadIdx.x, g = t >> 7, lane = t & 31, wt = t & 127;
  const int b = blockIdx.x / a.tiles_per_img;
  const int64_t p0 = (int64_t)(blockIdx.x - b * a.tiles_per_img) * BM;
  if (t == 0) {
    ptx::prefetch_tmap(&tmWt);
    ptx::mbar_init(&sm.full, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  if (t == 0) {                          // Wt pass 0 streams in during the prologue
    ptx::mbar_arrive_expect_tx(&sm.full, DOUT / BK * W_KB);
    for (int kb = 0; kb < DOUT / BK; ++kb) ptx::tma_load_2d(sm.wt[kb], &tmWt, &sm.full, kb * BK, 0);
  }
  // ---- prologue: four quarters of 32 pixels; warp = channels [32 grp, 32 grp + 32), lane = pixel ----
  {
    const int pr = t & 31, grp = t >> 5;
    const int64_t img = (int64_t)b * DOUT * a.HW;
    for (int qq = 0; qq < 4; ++qq) {
      const int r = 32 * qq + pr;
      const int64_t p = p0 + r;
      const bool pv = p < a.HW;
      float z[32], gy[32];
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int64_t o = img + (int64_t)(32 * grp + i) * a.HW + p;
        z[i] = pv ? to_f32(a.zn[o]) : 0.f;
        gy[i] = pv ? to_f32(a.gzn[o]) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) dot = fmaf(z[i], gy[i], dot);
      sm.red[grp][pr] = dot;
      __syncthreads();
      dot = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) dot += sm.red[k][pr];                                 // fixed order
      const float inv = pv ? a.inv_norm[(int64_t)b * a.HW + p] : 0.f;
      // d/dz [z / max(|z|, eps)] applied to gzn, with zn = z inv:  (gzn - zn <zn, gzn>) inv;  clamped: gzn inv
      const float coef = inv < NORM_EPS_INV ? dot : 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float gv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) gv[i] = (gy[8 * j + i] - z[8 * j + i] * coef) * inv;
        store8(sm.a[grp >> 1], r, 4 * (grp & 1) + j, gv);
        if (p < a.HWp) {
          __nv_bfloat16* dst = a.gz + ((int64_t)b * DOUT + 32 * grp + 8 * j) * a.HWp + p;
#pragma unroll
          for (int i = 0; i < 8; ++i) dst[(int64_t)i * a.HWp] = __float2bfloat16(gv[i]);
        }
      }
      __syncthreads();                   // sm.red is reused by the next quarter
    }
  }
  ptx::fence_proxy_async();
  __syncthreads();

  const int fr = 16 * (wt >> 5) + (lane >> 2), q = lane & 3;
  const uint32_t a_base = ptx::smem_u32(sm.a[0]) + g * WG_ROWS_BYTES, w_base = ptx::smem_u32(sm.wt[0]);
  T* gx = a.gx + (int64_t)b * a.Cin * a.HW;
  float acc[128];
  for (int np = 0; np < a.npass; ++np) {
    wait_full(&sm.full, (uint32_t)np & 1u);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < DOUT / 16; ++k)
      ptx::wgmma_m64n256k16<0>(acc, ptx::make_desc_kmajor_sw128(a_base + (k >> 2) * A_KB + (k & 3) * 32),
                               ptx::make_desc_kmajor_sw128(w_base + (k >> 2) * W_KB + (k & 3) * 32), k != 0 ? 1u : 0u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operands(acc);
    __syncthreads();                     // both warpgroups have read this pass's Wt
    if (t == 0 && np + 1 < a.npass) {
      ptx::mbar_arrive_expect_tx(&sm.full, DOUT / BK * W_KB);
      for (int kb = 0; kb < DOUT / BK; ++kb) ptx::tma_load_2d(sm.wt[kb], &tmWt, &sm.full, kb * BK, (np + 1) * DOUT);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t p = p0 + g * 64 + fr + 8 * h;
      if (p < a.HW) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = np * DOUT + 8 * i + 2 * q + e;
            if (c < a.Cin) gx[(int64_t)c * a.HW + p] = from_f32<T>(acc[4 * i + 2 * h + e]);
          }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
template <class T>
struct WgradArgs {
  const T* x; float* partials;
  int Cin, ldp; int64_t HW; int blk_per_img; int64_t units; int splits;
};

template <class T>
__global__ void __launch_bounds__(NT, 1) k_proj_wgrad(const __grid_constant__ CUtensorMap tmG, WgradArgs<T> a) {
  extern __shared__ uint8_t smem_raw[];
  WgradSmem& sm = aligned_smem<WgradSmem>(smem_raw);
  const int t = threadIdx.x, g = t >> 7, lane = t & 31, wt = t & 127;
  const int n0 = blockIdx.x * 128, c0 = blockIdx.y * DOUT, s = blockIdx.z;
  const int64_t u0 = a.units * s / a.splits, u1 = a.units * (s + 1) / a.splits;
  if (t == 0) {
    ptx::prefetch_tmap(&tmG);
    for (int i = 0; i < 3; ++i) ptx::mbar_init(&sm.full[i], 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  auto issue_a = [&](int64_t u, int stage) {
    const int bb = (int)(u / a.blk_per_img), pb = (int)(u - (int64_t)bb * a.blk_per_img);
    ptx::mbar_arrive_expect_tx(&sm.full[stage], A_KB);
    ptx::tma_load_2d(sm.a[stage], &tmG, &sm.full[stage], pb * WB, bb * DOUT + n0);
  };
  // conversion items: pixel row (t & 63) of the block, 16-byte channel chunks (t >> 6) + 4 j, j < 8 (32 chunks = 256 ch)
  const int pr = t & 63, cg = t >> 6;
  typename Staged<T>::type v[8][8];
  auto load_b = [&](int64_t u) {
    const int bb = (int)(u / a.blk_per_img), pb = (int)(u - (int64_t)bb * a.blk_per_img);
    const T* img = a.x + (int64_t)bb * a.Cin * a.HW;
#pragma unroll
    for (int j = 0; j < 8; ++j) load8(img, a.Cin, a.HW, c0 + 8 * (cg + 4 * j), (int64_t)pb * WB + pr, a.Cin, v[j]);
  };
  auto store_b = [&](int stage) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int chunk = cg + 4 * j;                     // 64-channel block chunk >> 3, 16-byte chunk chunk & 7
      store8(sm.b[stage] + (chunk >> 3) * (WB * 128), pr, chunk & 7, v[j]);
    }
  };
  if (t == 0)
    for (int i = 0; i < 2 && u0 + i < u1; ++i) issue_a(u0 + i, i);
  if (u0 < u1) {
    load_b(u0);
    store_b(0);
    ptx::fence_proxy_async();
  }
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  const uint32_t a_off = g * WG_ROWS_BYTES;
  for (int64_t u = u0; u < u1; ++u) {
    const int it = (int)(u - u0), sa = it % 3, sb = it & 1;
    __syncthreads();
    if (t == 0 && u + 2 < u1) issue_a(u + 2, (it + 2) % 3);
    const bool more = u + 1 < u1;
    if (more) load_b(u + 1);
    wait_full(&sm.full[sa], (uint32_t)(it / 3) & 1u);
    const uint32_t abase = ptx::smem_u32(sm.a[sa]) + a_off, bbase = ptx::smem_u32(sm.b[sb]);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < WB / 16; ++k)
      ptx::wgmma_m64n256k16<1>(acc, ptx::make_desc_kmajor_sw128(abase + k * 32),
                               ptx::make_desc_mnmajor_sw128(bbase + k * 2048, WB * 128, 1024), 1u);
    ptx::wgmma_commit();
    if (more) {
      store_b(sb ^ 1);
      ptx::fence_proxy_async();
    }
    ptx::wgmma_wait<0>();
    ptx::fence_operands(acc);
  }
  // partial (split s) rows n0 + 64 g + fr + 8 h, columns c0 + 8 i + 2 q
  const int fr = 16 * (wt >> 5) + (lane >> 2), q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* dst = a.partials + ((int64_t)s * DOUT + n0 + g * 64 + fr + 8 * h) * a.ldp + c0 + 2 * q;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
  }
}

__global__ void k_proj_reduce(const float* __restrict__ partials, int splits, int Cin, int ldp, float* __restrict__ gw,
                              float* __restrict__ gb) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)DOUT * (Cin + 1)) return;
  const int n = (int)(idx / (Cin + 1)), c = (int)(idx % (Cin + 1));
  float v = 0.f;
  for (int s = 0; s < splits; ++s) v += partials[((int64_t)s * DOUT + n) * ldp + c];     // fixed order
  if (c < Cin) gw[(int64_t)n * Cin + c] = v;
  else if (gb) gb[n] = v;
}

// ------------------------------------------------------------------------------------------------------------------
struct Layout {
  int cin64, cin256, ctiles, ldp;                // wgrad columns: Cin + 1 (the bias column) rounded up to 256
  int64_t HWp, wk_bytes, wt_off, pack_bytes;
  int64_t gz_bytes, part_off, scratch_bytes;
  int64_t units; int splits, blk_per_img;
};
static inline int64_t align1k(int64_t v) { return (v + 1023) & ~(int64_t)1023; }
static Layout layout(int B, int Cin, int64_t HW) {
  Layout L;
  L.cin64 = ceil_div(Cin, BK) * BK;
  L.cin256 = ceil_div(Cin, DOUT) * DOUT;
  L.ctiles = ceil_div(Cin + 1, DOUT);
  L.ldp = L.ctiles * DOUT;
  L.wk_bytes = align1k((int64_t)DOUT * L.cin64 * 2);
  L.wt_off = L.wk_bytes;
  L.pack_bytes = L.wt_off + align1k((int64_t)L.cin256 * DOUT * 2);
  L.HWp = ceil_div64(HW, WB) * WB;
  L.blk_per_img = (int)(L.HWp / WB);
  L.units = (int64_t)B * L.blk_per_img;
  const int mn = 2 * L.ctiles;
  int sp = num_sms() / mn;
  if (sp < 1) sp = 1;
  if ((int64_t)sp > L.units) sp = (int)L.units;
  L.splits = sp;
  L.gz_bytes = align1k((int64_t)B * DOUT * L.HWp * 2);
  L.part_off = L.gz_bytes;
  L.scratch_bytes = L.part_off + align1k((int64_t)L.splits * DOUT * L.ldp * 4);
  return L;
}
static inline bool shape_ok(int B, int Cin, int64_t HW) {
  return B > 0 && Cin > 0 && HW > 0 && (int64_t)B * DOUT * ceil_div64(HW, WB) * WB < (1ll << 40) &&
         ceil_div64(HW, BM) * B < (1ll << 31) && Cin <= (1 << 20);
}

}  // namespace proj
}  // namespace pcl

using namespace pcl;

namespace pcl { int tc_make_tmap_cols(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows); }

extern "C" int64_t pcl_proj_workspace_bytes(int32_t B, int32_t Cin, int64_t HW, int32_t which) {
  if (!proj::shape_ok(B, Cin, HW) || (which != 0 && which != 1)) return PCL_ERR_ARG;
  const proj::Layout L = proj::layout(B, Cin, HW);
  return which == 0 ? L.pack_bytes : L.scratch_bytes;
}

extern "C" int pcl_proj_pack(const float* weight, int32_t Cin, void* wpack, void* stream) {
  PCL_REQUIRE(weight && wpack && Cin > 0 && Cin <= (1 << 20));
  const proj::Layout L = proj::layout(1, Cin, 1);
  uint8_t* base = (uint8_t*)wpack;
  const int64_t n = (int64_t)proj::DOUT * L.cin256;
  proj::k_proj_pack<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(
      weight, Cin, L.cin64, L.cin256, (__nv_bfloat16*)base, (__nv_bfloat16*)(base + L.wt_off));
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

template <class T>
static int proj_fwd(const T* x, const void* wpack, const float* bias, int32_t B, int32_t Cin, int64_t HW, T* zn,
                    float* inv_norm, void* stream) {
  PCL_REQUIRE(x && wpack && zn && inv_norm && proj::shape_ok(B, Cin, HW));
  const proj::Layout L = proj::layout(B, Cin, HW);
  CUtensorMap tmW;
  int st = tc_make_tmap_cols(&tmW, wpack, (uint64_t)L.cin64, proj::DOUT, proj::DOUT);
  if (st != PCL_OK) return st;
  proj::FwdArgs<T> a;
  a.x = x; a.bias = bias; a.zn = zn; a.inv_norm = inv_norm;
  a.Cin = Cin; a.nkb = L.cin64 / proj::BK; a.HW = HW;
  a.tiles_per_img = (int)ceil_div64(HW, proj::BM);
  const size_t smem = sizeof(proj::FwdSmem) + 1024;
  PCL_SMEM_OPT_IN(proj::k_proj_fwd<T>, smem);
  proj::k_proj_fwd<T><<<(unsigned)(B * a.tiles_per_img), proj::NT, smem, (cudaStream_t)stream>>>(tmW, a);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_proj_fwd(const float* x, const void* wpack, const float* bias, int32_t B, int32_t Cin, int64_t HW,
                            float* zn, float* inv_norm, void* stream) {
  return pcl_proj_fwd_dt(x, PCL_DT_F32, wpack, bias, B, Cin, HW, zn, inv_norm, stream);
}

extern "C" int pcl_proj_fwd_dt(const void* x, int32_t dtype, const void* wpack, const float* bias, int32_t B,
                               int32_t Cin, int64_t HW, void* zn, float* inv_norm, void* stream) {
  if (dtype == PCL_DT_F32)
    return proj_fwd((const float*)x, wpack, bias, B, Cin, HW, (float*)zn, inv_norm, stream);
  if (dtype == PCL_DT_BF16)
    return proj_fwd((const __nv_bfloat16*)x, wpack, bias, B, Cin, HW, (__nv_bfloat16*)zn, inv_norm, stream);
  return PCL_ERR_ARG;                    // fp16 would be rounded to the bf16 GEMM operands: not offered
}

template <class T>
static int proj_bwd(const T* x, const T* zn, const float* inv_norm, const T* gzn, const void* wpack, int32_t B,
                    int32_t Cin, int64_t HW, void* scratch, T* gx, float* gw, float* gb, void* stream) {
  PCL_REQUIRE(x && zn && inv_norm && gzn && wpack && scratch && gx && gw && proj::shape_ok(B, Cin, HW));
  const proj::Layout L = proj::layout(B, Cin, HW);
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* sc = (uint8_t*)scratch;
  __nv_bfloat16* gz = (__nv_bfloat16*)sc;
  float* part = (float*)(sc + L.part_off);
  CUtensorMap tmWt, tmG;
  int st = tc_make_tmap_cols(&tmWt, (const uint8_t*)wpack + L.wt_off, proj::DOUT, (uint64_t)L.cin256, proj::DOUT);
  if (st != PCL_OK) return st;
  st = tc_make_tmap_cols(&tmG, gz, (uint64_t)L.HWp, (uint64_t)B * proj::DOUT, 128);
  if (st != PCL_OK) return st;

  proj::DgradArgs<T> d;
  d.zn = zn; d.gzn = gzn; d.inv_norm = inv_norm; d.gx = gx; d.gz = gz;
  d.Cin = Cin; d.npass = L.cin256 / proj::DOUT; d.HW = HW; d.HWp = L.HWp;
  d.tiles_per_img = (int)ceil_div64(HW, proj::BM);
  const size_t smem_d = sizeof(proj::DgradSmem) + 1024;
  PCL_SMEM_OPT_IN(proj::k_proj_dgrad<T>, smem_d);
  proj::k_proj_dgrad<T><<<(unsigned)(B * d.tiles_per_img), proj::NT, smem_d, s>>>(tmWt, d);
  PCL_LAUNCH_CHECK();

  proj::WgradArgs<T> w;
  w.x = x; w.partials = part; w.Cin = Cin; w.ldp = L.ldp; w.HW = HW; w.blk_per_img = L.blk_per_img;
  w.units = L.units; w.splits = L.splits;
  const size_t smem_w = sizeof(proj::WgradSmem) + 1024;
  PCL_SMEM_OPT_IN(proj::k_proj_wgrad<T>, smem_w);
  proj::k_proj_wgrad<T><<<dim3(proj::DOUT / 128, L.ctiles, L.splits), proj::NT, smem_w, s>>>(tmG, w);
  PCL_LAUNCH_CHECK();

  const int64_t n = (int64_t)proj::DOUT * (Cin + 1);
  proj::k_proj_reduce<<<(unsigned)ceil_div64(n, 256), 256, 0, s>>>(part, L.splits, Cin, L.ldp, gw, gb);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_proj_bwd(const float* x, const float* zn, const float* inv_norm, const float* gzn, const void* wpack,
                            int32_t B, int32_t Cin, int64_t HW, void* scratch, float* gx, float* gw, float* gb,
                            void* stream) {
  return pcl_proj_bwd_dt(x, PCL_DT_F32, zn, inv_norm, gzn, wpack, B, Cin, HW, scratch, gx, gw, gb, stream);
}

extern "C" int pcl_proj_bwd_dt(const void* x, int32_t dtype, const void* zn, const float* inv_norm, const void* gzn,
                               const void* wpack, int32_t B, int32_t Cin, int64_t HW, void* scratch, void* gx, float* gw,
                               float* gb, void* stream) {
  if (dtype == PCL_DT_F32)
    return proj_bwd((const float*)x, (const float*)zn, inv_norm, (const float*)gzn, wpack, B, Cin, HW, scratch,
                    (float*)gx, gw, gb, stream);
  if (dtype == PCL_DT_BF16)
    return proj_bwd((const __nv_bfloat16*)x, (const __nv_bfloat16*)zn, inv_norm, (const __nv_bfloat16*)gzn, wpack, B,
                    Cin, HW, scratch, (__nv_bfloat16*)gx, gw, gb, stream);
  return PCL_ERR_ARG;
}
