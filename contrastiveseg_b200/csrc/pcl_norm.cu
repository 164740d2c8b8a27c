// Projection head kernels.
// (1) L2 normalise over the channel dim of an NCHW tensor (SURVEY §8 row a1).
// Replaces lib/models/modules/projection.py:24  F.normalize(x, p=2, dim=1)  and its autograd backward.
// HBM-bound: forward reads x once and writes y once (2 * B*D*HW*4 bytes); backward reads x and gy once and
// writes gx once.  One CTA covers 32 consecutive pixels x all D channels: lanes run along the pixel
// dimension (coalesced 128 B rows), the 8 warps split the channels and keep their values in registers.
#include <type_traits>

#include "pcl_common.cuh"
#include "ptx_sm90.cuh"
#include "pcl_wgmma.cuh"

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
//   k_pack_bf16    W (256, Cin) fp32 -> Wk (256, Cin up to 64) bf16 and Wt (Cin up to 256, 256) bf16, zero-padded
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
struct WgradBnSmem : WgradSmem {
  alignas(16) float ss[2][DOUT];                 // scale, shift of the CTA's 256 channels (16-byte vector loads)
};
static_assert(sizeof(WgradBnSmem) + 1024 <= 227 * 1024, "shared memory of one H100 block");
struct DgradBnSmem : DgradSmem {
  float bnred[2][NT / 32][DOUT];                 // per-warp channel sums of g_u and g_u x_hat, one 256-channel pass
};
static_assert(sizeof(DgradBnSmem) + 1024 <= 227 * 1024, "shared memory of one H100 block");

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

// BatchNorm + ReLU in front of the GEMM (the BN = true instantiations).  `ss` is the per-channel state written by
// k_bn_finalize: scale at [0, ldp), shift at [ldp, 2 ldp), batch (or running) mean at [2 ldp, 3 ldp), invstd at
// [3 ldp, 4 ldp), 1 / count at 4 ldp.  ldp = the wgrad's column count (Cin + 1 rounded up to 256), so every channel any
// kernel converts has an entry: scale = shift = 0 beyond Cin, except scale = 1 at channel Cin, so the wgrad's constant-1
// bias channel passes through the affine unchanged (max(0, 1 * 1 + 0) = 1) and zero channels stay exactly 0.
struct BnPro {
  const float* ss; const void* y; float* part;   // y: the BN input (dgrad epilogue); part: per-tile sums (dgrad)
  int ldp;
};
template <class A> struct WithBn : A { BnPro bn; };
template <class A, bool BN> using ArgsBn = typename std::conditional<BN, WithBn<A>, A>::type;
template <class A> __device__ __forceinline__ BnPro bn_of(const A&) { return BnPro{nullptr, nullptr, nullptr, 0}; }
template <class A> __device__ __forceinline__ BnPro bn_of(const WithBn<A>& a) { return a.bn; }

__device__ __forceinline__ float raw_f32(float v) { return v; }
__device__ __forceinline__ float raw_f32(uint16_t v) { return __uint_as_float((uint32_t)v << 16); }

// u = max(0, y scale_c + shift_c) for channels [c, c + 8) in fp32; exactly 0 at pixels >= HW (pv false).  Runs at the
// tile store, after every raw load of the K-block has been issued.
template <class S>
__device__ __forceinline__ void bn_relu8(const S (&v)[8], const float* scale, const float* shift, bool pv,
                                         float (&u)[8]) {
  const float4* sc = reinterpret_cast<const float4*>(scale);
  const float4* sh = reinterpret_cast<const float4*>(shift);
  const float4 s0 = sc[0], s1 = sc[1], h0 = sh[0], h1 = sh[1];
  const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  const float h[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) u[i] = pv ? fmaxf(fmaf(raw_f32(v[i]), s[i], h[i]), 0.f) : 0.f;
}
// store8 of the staged activations, through the BatchNorm + ReLU when BN (scale at ss[c], shift at ss[ld + c])
template <bool BN, class S>
__device__ __forceinline__ void put8(uint8_t* tile, int r, int ch, const S (&v)[8], const float* ss, int ld, int c,
                                     bool pv) {
  if constexpr (BN) {
    float u[8];
    bn_relu8(v, ss + c, ss + ld + c, pv, u);
    store8(tile, r, ch, u);
  } else {
    store8(tile, r, ch, v);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// W (R, C) fp32 -> wk (ra, ca) = W and wt (rb, cb) = W^T in bf16, zero-padded (ra, cb >= R; ca, rb >= C).  Thread idx
// writes element idx of each (coalesced stores), so the grid covers the larger of the two.
__global__ void k_pack_bf16(const float* __restrict__ w, int R, int C, int ra, int ca, int rb, int cb,
                            __nv_bfloat16* __restrict__ wk, __nv_bfloat16* __restrict__ wt) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int r = (int)(idx / ca), c = (int)(idx % ca);
  if (idx < (int64_t)ra * ca) wk[idx] = __float2bfloat16(r < R && c < C ? w[(int64_t)r * C + c] : 0.f);
  if (idx < (int64_t)rb * cb) {
    if (cb != ca) { r = (int)(idx / cb); c = (int)(idx % cb); }   // equal widths (conv1): wk's 64-bit division
    wt[idx] = __float2bfloat16(r < C && c < R ? w[(int64_t)c * C + r] : 0.f);
  }
}

// ------------------------------------------------------------------------------------------------------------------
template <class T>
struct FwdArgs {
  const T* x; const float* bias; T* zn; float* inv_norm;
  int Cin, nkb; int64_t HW; int tiles_per_img;
};

// The K-loop of the forward-shaped GEMMs (k_proj_fwd, k_conv1_gemm): acc = the product of the activation tile (pixels
// p0 .. p0 + 127 of the NCHW image img, Cin channels) and rows n0 .. n0 + 255 of the K-major bf16 weight behind tmW,
// nkb K-blocks.  The threads convert the tile into the swizzled bf16 operand through put8<BN>, register-staged one
// K-block ahead; the weight comes by TMA in FWD_WSTAGES stages.  sm.bias[t] = bias_of(t), the bias of output channel
// n0 + t.
template <bool BN, class T, class BiasOf>
__device__ __forceinline__ void fwd_mainloop(FwdSmem& sm, const CUtensorMap& tmW, const T* img, int Cin, int64_t HW,
                                             int64_t p0, int n0, int nkb, BiasOf bias_of, const BnPro& bn,
                                             float (&acc)[128]) {
  const int t = threadIdx.x, g = t >> 7, wt = t & 127;
  if (t == 0) {
    ptx::prefetch_tmap(&tmW);
    for (int s = 0; s < FWD_WSTAGES; ++s) ptx::mbar_init(&sm.full[s], 1);
    ptx::fence_barrier_init();
  }
  sm.bias[t] = bias_of(t);
  __syncthreads();
  if (t == 0)
    for (int kb = 0; kb < 2 && kb < nkb; ++kb) {
      ptx::mbar_arrive_expect_tx(&sm.full[kb], W_KB);
      ptx::tma_load_2d(sm.w[kb], &tmW, &sm.full[kb], kb * BK, n0);
    }
  // conversion items of this thread: pixel row wt, 16-byte channel chunks g, g + 2, g + 4, g + 6 of each K-block
  typename Staged<T>::type v[4][8];
#pragma unroll
  for (int j = 0; j < 4; ++j) load8(img, Cin, HW, 8 * (g + 2 * j), p0 + wt, -1, v[j]);
#pragma unroll
  for (int j = 0; j < 4; ++j) put8<BN>(sm.a[0], wt, g + 2 * j, v[j], bn.ss, bn.ldp, 8 * (g + 2 * j), p0 + wt < HW);
  ptx::fence_proxy_async();

  const uint32_t a_off = g * WG_ROWS_BYTES;
  for (int kb = 0; kb < nkb; ++kb) {
    const int sa = kb & 1, sw = kb % FWD_WSTAGES;
    __syncthreads();                     // A[sa] complete; every wgmma of K-block kb - 1 retired (stage reuse below)
    if (t == 0 && kb + 2 < nkb) {
      const int s2 = (kb + 2) % FWD_WSTAGES;
      ptx::mbar_arrive_expect_tx(&sm.full[s2], W_KB);
      ptx::tma_load_2d(sm.w[s2], &tmW, &sm.full[s2], (kb + 2) * BK, n0);
    }
    const bool more = kb + 1 < nkb;
    if (more) {
#pragma unroll
      for (int j = 0; j < 4; ++j) load8(img, Cin, HW, (kb + 1) * BK + 8 * (g + 2 * j), p0 + wt, -1, v[j]);
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
      for (int j = 0; j < 4; ++j)
        put8<BN>(sm.a[sa ^ 1], wt, g + 2 * j, v[j], bn.ss, bn.ldp, (kb + 1) * BK + 8 * (g + 2 * j), p0 + wt < HW);
      ptx::fence_proxy_async();
    }
    ptx::wgmma_wait<0>();
    ptx::fence_operands(acc);
  }
}

template <class T, bool BN = false>
__global__ void __launch_bounds__(NT, 1) k_proj_fwd(const __grid_constant__ CUtensorMap tmW, ArgsBn<FwdArgs<T>, BN> a) {
  extern __shared__ uint8_t smem_raw[];
  FwdSmem& sm = aligned_smem<FwdSmem>(smem_raw);
  const int t = threadIdx.x, g = t >> 7, lane = t & 31, wt = t & 127;
  const int b = blockIdx.x / a.tiles_per_img;
  const int64_t p0 = (int64_t)(blockIdx.x - b * a.tiles_per_img) * BM;
  float acc[128];
  fwd_mainloop<BN>(sm, tmW, a.x + (int64_t)b * a.Cin * a.HW, a.Cin, a.HW, p0, 0, a.nkb,
                   [&](int c) { return a.bias ? a.bias[c] : 0.f; }, bn_of(a), acc);

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

template <class T, bool BN = false>
__global__ void __launch_bounds__(NT, 1) k_proj_dgrad(const __grid_constant__ CUtensorMap tmWt,
                                                      ArgsBn<DgradArgs<T>, BN> a) {
  extern __shared__ uint8_t smem_raw[];
  using Smem = typename std::conditional<BN, DgradBnSmem, DgradSmem>::type;
  Smem& sm = aligned_smem<Smem>(smem_raw);
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
    if constexpr (BN) {
      // acc is g_a, the gradient of the ReLU output.  g_u = g_a [y scale + shift > 0] (the forward's test) goes to gx;
      // this tile's per-channel sums of g_u and g_u x_hat, x_hat = (y - mean) invstd, go to the partials, reduced in a
      // fixed order: over the warp's 16 pixels by shuffles, over the 8 warps through shared memory.
      const BnPro bn = a.bn;
      const T* y = static_cast<const T*>(bn.y) + (int64_t)b * a.Cin * a.HW;
#pragma unroll
      for (int i = 0; i < 32; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int cl = 8 * i + 2 * q + e, c = np * DOUT + cl;
          const float sc = bn.ss[c], sh = bn.ss[bn.ldp + c], mu = bn.ss[2 * bn.ldp + c], is = bn.ss[3 * bn.ldp + c];
          float yv[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t p = p0 + g * 64 + fr + 8 * h;
            yv[h] = (p < a.HW && c < a.Cin) ? to_f32(y[(int64_t)c * a.HW + p]) : 0.f;
          }
          float s1 = 0.f, s2 = 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t p = p0 + g * 64 + fr + 8 * h;
            if (p < a.HW && c < a.Cin) {
              const float gu = fmaf(yv[h], sc, sh) > 0.f ? acc[4 * i + 2 * h + e] : 0.f;
              gx[(int64_t)c * a.HW + p] = from_f32<T>(gu);
              s1 += gu;
              s2 = fmaf(gu, (yv[h] - mu) * is, s2);
            }
          }
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) {
            s1 += __shfl_xor_sync(0xffffffffu, s1, m);
            s2 += __shfl_xor_sync(0xffffffffu, s2, m);
          }
          if (lane < 4) {
            sm.bnred[0][t >> 5][cl] = s1;
            sm.bnred[1][t >> 5][cl] = s2;
          }
        }
      __syncthreads();                   // bnred is rewritten by the next pass only after its post-wgmma barrier
      float r1 = 0.f, r2 = 0.f;
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) { r1 += sm.bnred[0][w][t]; r2 += sm.bnred[1][w][t]; }     // fixed order
      float* part = bn.part + (int64_t)blockIdx.x * 2 * bn.ldp + np * DOUT + t;
      part[0] = r1;
      part[bn.ldp] = r2;
    } else {
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
}

// ------------------------------------------------------------------------------------------------------------------
template <class T>
struct WgradArgs {
  const T* x; float* partials;
  int Cin, ldp; int64_t HW; int blk_per_img; int64_t units; int splits;
};

template <class T, bool BN = false>
__global__ void __launch_bounds__(NT, 1) k_proj_wgrad(const __grid_constant__ CUtensorMap tmG, ArgsBn<WgradArgs<T>, BN> a) {
  extern __shared__ uint8_t smem_raw[];
  using Smem = typename std::conditional<BN, WgradBnSmem, WgradSmem>::type;
  Smem& sm = aligned_smem<Smem>(smem_raw);
  const int t = threadIdx.x, g = t >> 7, lane = t & 31, wt = t & 127;
  const int n0 = blockIdx.x * 128, c0 = blockIdx.y * DOUT, s = blockIdx.z;
  const int64_t u0 = a.units * s / a.splits, u1 = a.units * (s + 1) / a.splits;
  if (t == 0) {
    ptx::prefetch_tmap(&tmG);
    for (int i = 0; i < 3; ++i) ptx::mbar_init(&sm.full[i], 1);
    ptx::fence_barrier_init();
  }
  const float* sss = nullptr;                           // BN: scale / shift of this CTA's 256 channels
  if constexpr (BN) {
    const BnPro bn = a.bn;
    sm.ss[0][t] = bn.ss[c0 + t];
    sm.ss[1][t] = bn.ss[bn.ldp + c0 + t];
    sss = sm.ss[0];
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
  bool pvb = false;                                     // BN: the staged pixel is < HW
  auto load_b = [&](int64_t u) {
    const int bb = (int)(u / a.blk_per_img), pb = (int)(u - (int64_t)bb * a.blk_per_img);
    const T* img = a.x + (int64_t)bb * a.Cin * a.HW;
    if constexpr (BN) pvb = (int64_t)pb * WB + pr < a.HW;
#pragma unroll
    for (int j = 0; j < 8; ++j) load8(img, a.Cin, a.HW, c0 + 8 * (cg + 4 * j), (int64_t)pb * WB + pr, a.Cin, v[j]);
  };
  auto store_b = [&](int stage) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int chunk = cg + 4 * j;                     // 64-channel block chunk >> 3, 16-byte chunk chunk & 7
      put8<BN>(sm.b[stage] + (chunk >> 3) * (WB * 128), pr, chunk & 7, v[j], sss, DOUT, 8 * chunk, pvb);
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

// rows n < `rows` of the partials -> gw (rows, Cin) and gb (rows)
__global__ void k_proj_reduce(const float* __restrict__ partials, int splits, int rows, int Cin, int ldp,
                              float* __restrict__ gw, float* __restrict__ gb) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)rows * (Cin + 1)) return;
  const int n = (int)(idx / (Cin + 1)), c = (int)(idx % (Cin + 1));
  float v = 0.f;
  for (int s = 0; s < splits; ++s) v += partials[((int64_t)s * DOUT + n) * ldp + c];     // fixed order
  if (c < Cin) gw[(int64_t)n * Cin + c] = v;
  else if (gb) gb[n] = v;
}

// ------------------------------------------------------------------------------------------------------------------
// BatchNorm statistics of y (B, C, HW), one CTA per channel: sum y and sum y^2 in fp64 (y^2 of an fp32 value is exact in
// fp64, so var = E[y^2] - E[y]^2 keeps ~1e-16 relative accuracy where fp32 would cancel), in a fixed order (per-thread
// strided sums, then a fixed shuffle tree and a fixed-order sum over the warps): bit-reproducible.  fp64 sums add up
// across ranks, so SyncBatchNorm all-reduces them as they are.  sums[C + c] = sum y^2, sums[2 C] = B * HW.
constexpr int ST_NT = 256, ST_UNROLL = 8;
template <class T>
__global__ void __launch_bounds__(ST_NT) k_bn_stats(const T* __restrict__ y, int B, int C, int64_t HW,
                                                     double* __restrict__ sums) {
  __shared__ double red[2][ST_NT / 32];
  const int c = blockIdx.x, t = threadIdx.x;
  double s = 0., s2 = 0.;
  for (int b = 0; b < B; ++b) {
    const T* row = y + ((int64_t)b * C + c) * HW;
    for (int64_t p0 = 0; p0 < HW; p0 += (int64_t)ST_NT * ST_UNROLL) {
      float v[ST_UNROLL];
#pragma unroll
      for (int k = 0; k < ST_UNROLL; ++k) {             // every load of the batch before any arithmetic
        const int64_t p = p0 + k * ST_NT + t;
        v[k] = p < HW ? to_f32(row[p]) : 0.f;
      }
#pragma unroll
      for (int k = 0; k < ST_UNROLL; ++k) {
        const double d = v[k];
        s += d;
        s2 = fma(d, d, s2);
      }
    }
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, m);
    s2 += __shfl_xor_sync(0xffffffffu, s2, m);
  }
  if ((t & 31) == 0) { red[0][t >> 5] = s; red[1][t >> 5] = s2; }
  __syncthreads();
  if (t == 0) {
    double r = 0., r2 = 0.;
    for (int w = 0; w < ST_NT / 32; ++w) { r += red[0][w]; r2 += red[1][w]; }
    sums[c] = r;
    sums[C + c] = r2;
    if (c == 0) sums[2 * C] = (double)B * (double)HW;
  }
}

// sums (or the running buffers) -> the per-channel state of BnPro; training: running buffers updated in place as
// nn.BatchNorm2d does (momentum, unbiased variance over the global count)
__global__ void k_bn_finalize(const double* __restrict__ sums, const float* __restrict__ gamma,
                              const float* __restrict__ beta, float* __restrict__ rmean, float* __restrict__ rvar, int C,
                              int ldp, float eps, float momentum, int training, float* __restrict__ st) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ldp) return;
  float scale = c == C ? 1.f : 0.f, shift = 0.f, mean = 0.f, invstd = 0.f;
  if (c < C) {
    double m, var;
    if (training) {
      const double n = sums[2 * C];
      m = sums[c] / n;
      var = fmax(sums[C + c] / n - m * m, 0.);
      rmean[c] = (float)((1. - momentum) * rmean[c] + momentum * m);
      rvar[c] = (float)((1. - momentum) * rvar[c] + momentum * var * n / (n - 1.));
    } else {
      m = rmean[c];
      var = rvar[c];
    }
    invstd = (float)(1. / sqrt(var + (double)eps));
    mean = (float)m;
    scale = gamma[c] * invstd;
    shift = beta[c] - mean * scale;
  }
  st[c] = scale;
  st[ldp + c] = shift;
  st[2 * ldp + c] = mean;
  st[3 * ldp + c] = invstd;
  if (c == 0) st[4 * ldp] = training ? (float)(1. / sums[2 * C]) : 0.f;
}

// Per-tile, per-channel sum pairs part [tile][2][ld] -> sums[c], sums[C + c] in a fixed order: 32 channels per block,
// the 32 warps stride the tiles, then a fixed-order sum over the warps.  Used for the dgrad epilogue's sums of g_u and
// g_u x_hat (float; copy1 / copy2 = gbeta / ggamma, may be null) and for conv1's fp64 statistics of y (count > 0 goes
// to sums[2 C]).
constexpr int TS_NT = 1024;
template <class S>
__global__ void __launch_bounds__(TS_NT) k_tile_sum(const S* __restrict__ part, int64_t ntiles, int C, int ld,
                                                    S* __restrict__ sums, S* __restrict__ copy1, S* __restrict__ copy2,
                                                    double count) {
  __shared__ S red[2][TS_NT / 32][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, c = blockIdx.x * 32 + lane;
  S s1 = 0, s2 = 0;
  if (c < C)
    for (int64_t tile = w; tile < ntiles; tile += TS_NT / 32) {
      s1 += part[tile * 2 * ld + c];
      s2 += part[(tile * 2 + 1) * ld + c];
    }
  red[0][w][lane] = s1;
  red[1][w][lane] = s2;
  __syncthreads();
  if (w == 0 && c < C) {
    S r1 = 0, r2 = 0;
    for (int k = 0; k < TS_NT / 32; ++k) { r1 += red[0][k][lane]; r2 += red[1][k][lane]; }
    sums[c] = r1;
    sums[C + c] = r2;
    if (copy1) copy1[c] = r1;
    if (copy2) copy2[c] = r2;
    if (c == 0 && count > 0) sums[2 * C] = count;
  }
}

// BatchNorm input gradient, in place over g (= g_u in, g_y out): training g_y = scale (g_u - mean(g_u) - x_hat
// mean(g_u x_hat)) with the means over the (global) count; eval g_y = scale g_u.  scale = gamma invstd.
constexpr int IG_NT = 256, IG_UNROLL = 8;
template <class T>
__global__ void __launch_bounds__(IG_NT) k_bn_input_grad(const T* __restrict__ y, T* __restrict__ g,
                                                          const float* __restrict__ st, const float* __restrict__ gsum,
                                                          int C, int ldp, int64_t HW, int training) {
  const int64_t row = blockIdx.x;                       // b * C + c
  const int c = (int)(row % C);
  const float a = st[c], mu = st[2 * ldp + c], is = st[3 * ldp + c];
  float k1 = 0.f, k2 = 0.f;
  if (training) {
    const float invn = st[4 * ldp];
    k1 = gsum[c] * invn;
    k2 = gsum[C + c] * invn * is;
  }
  const int64_t p0 = (int64_t)blockIdx.y * IG_NT * IG_UNROLL + threadIdx.x;
  const T* yr = y + row * HW;
  T* gr = g + row * HW;
  float yv[IG_UNROLL], gv[IG_UNROLL];
#pragma unroll
  for (int k = 0; k < IG_UNROLL; ++k) {
    const int64_t p = p0 + k * IG_NT;
    yv[k] = p < HW ? to_f32(yr[p]) : 0.f;
    gv[k] = p < HW ? to_f32(gr[p]) : 0.f;
  }
#pragma unroll
  for (int k = 0; k < IG_UNROLL; ++k) {
    const int64_t p = p0 + k * IG_NT;
    if (p < HW) gr[p] = from_f32<T>(a * (gv[k] - k1 - (yv[k] - mu) * k2));
  }
}

// ------------------------------------------------------------------------------------------------------------------
struct Layout {
  int cin64, cin256, ctiles, ldp;                // wgrad columns: Cin + 1 (the bias column) rounded up to 256
  int64_t HWp, wk_bytes, wt_off, pack_bytes;
  int64_t gz_bytes, part_off, scratch_bytes;
  int64_t units; int splits, blk_per_img;
  int64_t ntiles, bn_part_off, bn_scratch_bytes, bn_state_bytes;   // BatchNorm + ReLU variant
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
  L.ntiles = (int64_t)B * ceil_div64(HW, BM);
  L.bn_part_off = L.scratch_bytes;
  L.bn_scratch_bytes = L.bn_part_off + align1k(L.ntiles * 2 * L.ldp * 4);
  L.bn_state_bytes = align1k(((int64_t)4 * L.ldp + 4) * 4);
  return L;
}
static inline bool shape_ok(int B, int Cin, int64_t HW) {
  return B > 0 && Cin > 0 && HW > 0 && (int64_t)B * DOUT * ceil_div64(HW, WB) * WB < (1ll << 40) &&
         ceil_div64(HW, BM) * B < (1ll << 31) && Cin <= (1 << 20);
}

// ------------------------------------------------------------------------------------------------------------------
// (4) The head's first 1x1 convolution, C -> C, in front of (3) (ProjectionHead(..., fuse_conv1=True)).
// Replaces lib/models/modules/projection.py:17-19's Conv2d(dim_in, dim_in, 1), its autograd backward and (3)'s
// statistics pass over y.  bf16 operands, fp32 accumulate, as (2).
//   k_pack_bf16      W1 (C, C) fp32 -> W1 and W1^T bf16, each (C up to 256 rows, C up to 64 columns), zero-padded
//   k_conv1_gemm     out = W . a per pixel: CTA = 128 pixels of one image x one 256-channel band of the output; A = the
//                    activation tile converted by the threads, B = the band's 256 rows of W by TMA (k_proj_fwd's loop).
//                    The bands of one pixel tile are consecutive CTAs, so the tile is read from HBM about once and
//                    from L2 by its other bands.  The epilogue stages the tile [channel][pixel] in the retired weight
//                    stages (two halves of 128 channels) and writes it along pixels.
//                    Forward (W1, x -> y): + b1, and per tile and channel the fp64 sums of the stored y and y^2 (the
//                    values as rounded to y's type), over 32 lanes by a fixed shuffle tree.
//                    Data gradient (W1^T, g_y -> gx).
//   k_tile_sum<double>  per-tile sums -> sums[2 C + 1] in pcl_proj_bn_stats_dt's layout (fp64, fixed order)
//   k_conv1_gy_pack  g_y -> bf16 in 256-row bands [band][b][256][HW up to 64], zero-padded: the TMA operand of
//   k_proj_wgrad, k_proj_reduce  run once per band of gW1's rows, reduced straight into the band's rows of gW1; the
//                    band's gb1 comes from the constant-1 channel.
struct Conv1Layout {
  int kp, np, nbands, tiles_per_img;             // K padded to 64, rows padded to 256 = nbands x 256
  int64_t ptiles, wt_off, pack_bytes, fwd_bytes;
  int64_t gy_bytes, part_off, bwd_bytes;
  Layout w;                                      // the weight gradient's pixel blocks and split-K partials
};
static Conv1Layout conv1_layout(int B, int C, int64_t HW) {
  Conv1Layout L;
  L.kp = ceil_div(C, BK) * BK;
  L.nbands = ceil_div(C, DOUT);
  L.np = L.nbands * DOUT;
  L.tiles_per_img = (int)ceil_div64(HW, BM);
  L.ptiles = (int64_t)B * L.tiles_per_img;
  L.wt_off = align1k((int64_t)L.np * L.kp * 2);
  L.pack_bytes = 2 * L.wt_off;
  L.fwd_bytes = align1k(L.ptiles * 2 * L.np * 8);
  L.w = layout(B, C, HW);
  L.gy_bytes = align1k((int64_t)L.np * B * L.w.HWp * 2);
  L.part_off = L.gy_bytes;
  L.bwd_bytes = L.part_off + align1k((int64_t)L.w.splits * DOUT * L.w.ldp * 4);
  return L;
}
constexpr int GP_NT = 256, GP_UNROLL = 8;
static inline bool conv1_shape_ok(int B, int C, int64_t HW) {
  if (!shape_ok(B, C, HW)) return false;
  const int64_t nb = ceil_div(C, DOUT), HWp = ceil_div64(HW, WB) * WB;
  return ceil_div64(HW, BM) * B * nb < (1ll << 31) && (int64_t)B * nb * DOUT < (1ll << 31) &&
         ceil_div64(HWp, (int64_t)GP_NT * GP_UNROLL) <= 65535;
}

template <class T>
struct Conv1Args {
  const T* a; const float* bias; T* out; double* part;   // bias, part (per-tile sums) may be null
  int C, nkb, nbands, np; int64_t HW; int tiles_per_img;
};

template <class T>
__global__ void __launch_bounds__(NT, 1) k_conv1_gemm(const __grid_constant__ CUtensorMap tmW, Conv1Args<T> a) {
  extern __shared__ uint8_t smem_raw[];
  FwdSmem& sm = aligned_smem<FwdSmem>(smem_raw);
  const int t = threadIdx.x, g = t >> 7, lane = t & 31, wt = t & 127;
  const int band = blockIdx.x % a.nbands, tile = blockIdx.x / a.nbands;
  const int b = tile / a.tiles_per_img, n0 = band * DOUT;
  const int64_t p0 = (int64_t)(tile - b * a.tiles_per_img) * BM;
  float acc[128];
  fwd_mainloop<false>(sm, tmW, a.a + (int64_t)b * a.C * a.HW, a.C, a.HW, p0, n0, a.nkb,
                      [&](int c) { return (a.bias && n0 + c < a.C) ? a.bias[n0 + c] : 0.f; }, BnPro{}, acc);

  // epilogue: acc[4 i + 2 h + e] = pixel g 64 + fr + 8 h of the tile, channel n0 + 8 i + 2 q + e.  Staging pitch LD (in
  // elements): a fragment store's 8 pixel rows x 4 channel pairs fall on distinct banks (132 words; 68 words for 2-byte T).
  const int fr = 16 * (wt >> 5) + (lane >> 2), q = lane & 3;
  constexpr int HALF = DOUT / 2, LD = sizeof(T) == 4 ? BM + 4 : BM + 8;
  static_assert(HALF * LD * sizeof(T) <= sizeof(FwdSmem::w), "half a staged tile fits the weight stages");
  T* stage = reinterpret_cast<T*>(sm.w[0]);
  T* out = a.out + (int64_t)b * a.C * a.HW;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    __syncthreads();                     // hh 0: every wgmma has read sm.w; hh 1: the first half is written out
#pragma unroll
    for (int i = 0; i < HALF / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int cl = 8 * i + 2 * q + e;
          stage[cl * LD + g * 64 + fr + 8 * h] = from_f32<T>(acc[4 * (HALF / 8 * hh + i) + 2 * h + e] +
                                                             sm.bias[HALF * hh + cl]);
        }
    __syncthreads();
    for (int cl = t >> 5; cl < HALF; cl += NT / 32) {          // warp = channel row, lane = pixel
      const int c = n0 + HALF * hh + cl;
      if (c >= a.C) break;
      double s = 0., s2 = 0.;
#pragma unroll
      for (int j = 0; j < BM / 32; ++j) {
        const int px = 32 * j + lane;
        if (p0 + px < a.HW) {
          const T v = stage[cl * LD + px];
          out[(int64_t)c * a.HW + p0 + px] = v;
          const double d = to_f32(v);
          s += d;
          s2 = fma(d, d, s2);
        }
      }
      if (a.part) {
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
          s += __shfl_xor_sync(0xffffffffu, s, m);
          s2 += __shfl_xor_sync(0xffffffffu, s2, m);
        }
        if (lane == 0) {
          a.part[(int64_t)tile * 2 * a.np + c] = s;
          a.part[((int64_t)tile * 2 + 1) * a.np + c] = s2;
        }
      }
    }
  }
}

// g_y (B, C, HW) -> bf16 [band][b][256][HWp]: block row = (band B + b) 256 + r, zeros beyond C and HW
template <class T>
__global__ void __launch_bounds__(GP_NT) k_conv1_gy_pack(const T* __restrict__ gy, int B, int C, int64_t HW,
                                                         int64_t HWp, __nv_bfloat16* __restrict__ out) {
  const int64_t row = blockIdx.x;
  const int r = (int)(row % DOUT), bb = (int)(row / DOUT);
  const int b = bb % B, c = (bb / B) * DOUT + r;
  const T* src = gy + ((int64_t)b * C + c) * HW;
  __nv_bfloat16* dst = out + row * HWp;
  const int64_t p0 = (int64_t)blockIdx.y * GP_NT * GP_UNROLL + threadIdx.x;
  float v[GP_UNROLL];
#pragma unroll
  for (int k = 0; k < GP_UNROLL; ++k) {
    const int64_t p = p0 + k * GP_NT;
    v[k] = (c < C && p < HW) ? to_f32(src[p]) : 0.f;
  }
#pragma unroll
  for (int k = 0; k < GP_UNROLL; ++k) {
    const int64_t p = p0 + k * GP_NT;
    if (p < HWp) dst[p] = __float2bfloat16(v[k]);
  }
}

}  // namespace proj
}  // namespace pcl

using namespace pcl;

extern "C" int64_t pcl_proj_workspace_bytes(int32_t B, int32_t Cin, int64_t HW, int32_t which) {
  if (!proj::shape_ok(B, Cin, HW) || (which != 0 && which != 1)) return PCL_ERR_ARG;
  const proj::Layout L = proj::layout(B, Cin, HW);
  return which == 0 ? L.pack_bytes : L.scratch_bytes;
}

extern "C" int pcl_proj_pack(const float* weight, int32_t Cin, void* wpack, void* stream) {
  PCL_REQUIRE(weight && wpack && Cin > 0 && Cin <= (1 << 20));
  const proj::Layout L = proj::layout(1, Cin, 1);
  uint8_t* base = (uint8_t*)wpack;
  const int64_t n = (int64_t)proj::DOUT * L.cin256;                 // Wt's elements, >= Wk's
  proj::k_pack_bf16<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(
      weight, proj::DOUT, Cin, proj::DOUT, L.cin64, L.cin256, proj::DOUT, (__nv_bfloat16*)base,
      (__nv_bfloat16*)(base + L.wt_off));
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

template <class T, bool BN = false>
static int proj_fwd(const T* x, const void* wpack, const float* bias, int32_t B, int32_t Cin, int64_t HW, T* zn,
                    float* inv_norm, void* stream, proj::BnPro bn = {}) {
  PCL_REQUIRE(x && wpack && zn && inv_norm && proj::shape_ok(B, Cin, HW));
  const proj::Layout L = proj::layout(B, Cin, HW);
  CUtensorMap tmW;
  int st = tc_make_tmap(&tmW, wpack, (uint64_t)L.cin64, proj::DOUT, proj::DOUT);
  if (st != PCL_OK) return st;
  proj::ArgsBn<proj::FwdArgs<T>, BN> a;
  a.x = x; a.bias = bias; a.zn = zn; a.inv_norm = inv_norm;
  a.Cin = Cin; a.nkb = L.cin64 / proj::BK; a.HW = HW;
  a.tiles_per_img = (int)ceil_div64(HW, proj::BM);
  if constexpr (BN) a.bn = bn;
  const size_t smem = sizeof(proj::FwdSmem) + 1024;
  PCL_SMEM_OPT_IN((proj::k_proj_fwd<T, BN>), smem);
  proj::k_proj_fwd<T, BN><<<(unsigned)(B * a.tiles_per_img), proj::NT, smem, (cudaStream_t)stream>>>(tmW, a);
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

// Weight gradient of the bf16 gz rows [b][256][HWp] against x (L = layout(B, Cin, HW)): split-K partials, then the
// fixed-order reduce of their first `rows` rows into gw (rows, Cin) and gb (rows; may be null).
template <class T, bool BN>
static int proj_wgrad(const __nv_bfloat16* gz, const T* x, int32_t B, int32_t Cin, int64_t HW, const proj::Layout& L,
                      float* part, int rows, float* gw, float* gb, proj::BnPro bn, cudaStream_t s) {
  CUtensorMap tmG;
  const int st = tc_make_tmap(&tmG, gz, (uint64_t)L.HWp, (uint64_t)B * proj::DOUT, 128);
  if (st != PCL_OK) return st;
  proj::ArgsBn<proj::WgradArgs<T>, BN> w;
  w.x = x; w.partials = part; w.Cin = Cin; w.ldp = L.ldp; w.HW = HW; w.blk_per_img = L.blk_per_img;
  w.units = L.units; w.splits = L.splits;
  if constexpr (BN) w.bn = bn;
  const size_t smem_w = (BN ? sizeof(proj::WgradBnSmem) : sizeof(proj::WgradSmem)) + 1024;
  PCL_SMEM_OPT_IN((proj::k_proj_wgrad<T, BN>), smem_w);
  proj::k_proj_wgrad<T, BN><<<dim3(proj::DOUT / 128, L.ctiles, L.splits), proj::NT, smem_w, s>>>(tmG, w);
  PCL_LAUNCH_CHECK();
  const int64_t n = (int64_t)rows * (Cin + 1);
  proj::k_proj_reduce<<<(unsigned)ceil_div64(n, 256), 256, 0, s>>>(part, L.splits, rows, Cin, L.ldp, gw, gb);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

template <class T, bool BN = false>
static int proj_bwd(const T* x, const T* zn, const float* inv_norm, const T* gzn, const void* wpack, int32_t B,
                    int32_t Cin, int64_t HW, void* scratch, T* gx, float* gw, float* gb, void* stream,
                    proj::BnPro bn = {}) {
  PCL_REQUIRE(x && zn && inv_norm && gzn && wpack && scratch && gx && gw && proj::shape_ok(B, Cin, HW));
  const proj::Layout L = proj::layout(B, Cin, HW);
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* sc = (uint8_t*)scratch;
  __nv_bfloat16* gz = (__nv_bfloat16*)sc;
  CUtensorMap tmWt;
  const int st = tc_make_tmap(&tmWt, (const uint8_t*)wpack + L.wt_off, proj::DOUT, (uint64_t)L.cin256, proj::DOUT);
  if (st != PCL_OK) return st;

  proj::ArgsBn<proj::DgradArgs<T>, BN> d;
  d.zn = zn; d.gzn = gzn; d.inv_norm = inv_norm; d.gx = gx; d.gz = gz;
  d.Cin = Cin; d.npass = L.cin256 / proj::DOUT; d.HW = HW; d.HWp = L.HWp;
  d.tiles_per_img = (int)ceil_div64(HW, proj::BM);
  if constexpr (BN) d.bn = bn;
  const size_t smem_d = (BN ? sizeof(proj::DgradBnSmem) : sizeof(proj::DgradSmem)) + 1024;
  PCL_SMEM_OPT_IN((proj::k_proj_dgrad<T, BN>), smem_d);
  proj::k_proj_dgrad<T, BN><<<(unsigned)(B * d.tiles_per_img), proj::NT, smem_d, s>>>(tmWt, d);
  PCL_LAUNCH_CHECK();
  return proj_wgrad<T, BN>(gz, x, B, Cin, HW, L, (float*)(sc + L.part_off), proj::DOUT, gw, gb, bn, s);
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

// (3) BatchNorm2d / SyncBatchNorm + ReLU in front of the fused last conv (ProjectionHead(fused=True, fuse_bn_relu=True)).
// Replaces lib/models/modules/projection.py:17-24's BN and ReLU: the statistics pass reads y once, the GEMMs apply
// max(0, y scale + shift) where they convert the activation tile, the dgrad epilogue masks g_a by the ReLU and sums the
// BN backward's per-channel terms, and one elementwise pass forms the input gradient.
//   k_bn_stats        fp64 sum y, sum y^2 per channel (one CTA per channel, fixed order)
//   k_bn_finalize     -> scale, shift, mean, invstd (+ running buffers in training)
//   k_proj_fwd<T, true>, k_proj_dgrad<T, true>, k_proj_wgrad<T, true>   the GEMMs with the BN + ReLU prologue / epilogue
//   k_tile_sum<float>  per-tile sums of the dgrad epilogue -> sum g_u, sum g_u x_hat (fixed order)
//   k_bn_input_grad   g_u -> g_y in place
extern "C" int64_t pcl_proj_bn_workspace_bytes(int32_t B, int32_t Cin, int64_t HW, int32_t which) {
  if (!proj::shape_ok(B, Cin, HW) || (which != 0 && which != 1)) return PCL_ERR_ARG;
  const proj::Layout L = proj::layout(B, Cin, HW);
  return which == 0 ? L.bn_state_bytes : L.bn_scratch_bytes;
}

static inline bool bn_dtype_ok(int32_t dtype) { return dtype == PCL_DT_F32 || dtype == PCL_DT_BF16; }
static inline bool bn_shape_ok(int32_t B, int32_t Cin, int64_t HW) {
  return proj::shape_ok(B, Cin, HW) && (int64_t)B * Cin < (1ll << 31) &&
         ceil_div64(HW, (int64_t)proj::IG_NT * proj::IG_UNROLL) <= 65535;
}

extern "C" int pcl_proj_bn_stats_dt(const void* y, int32_t dtype, int32_t B, int32_t Cin, int64_t HW, double* sums,
                                    void* stream) {
  PCL_REQUIRE(y && sums && bn_dtype_ok(dtype) && bn_shape_ok(B, Cin, HW));
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == PCL_DT_F32)
    proj::k_bn_stats<float><<<(unsigned)Cin, proj::ST_NT, 0, s>>>((const float*)y, B, Cin, HW, sums);
  else
    proj::k_bn_stats<__nv_bfloat16><<<(unsigned)Cin, proj::ST_NT, 0, s>>>((const __nv_bfloat16*)y, B, Cin, HW, sums);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_proj_bn_finalize(const double* sums, const float* gamma, const float* beta, float* running_mean,
                                    float* running_var, int32_t Cin, float eps, float momentum, int32_t training,
                                    void* bn_state, void* stream) {
  PCL_REQUIRE(gamma && beta && running_mean && running_var && bn_state && Cin > 0 && Cin <= (1 << 20) && eps >= 0.f);
  PCL_REQUIRE(training == 0 || (training == 1 && sums));
  const proj::Layout L = proj::layout(1, Cin, 1);
  proj::k_bn_finalize<<<(unsigned)ceil_div(L.ldp, 256), 256, 0, (cudaStream_t)stream>>>(
      sums, gamma, beta, running_mean, running_var, Cin, L.ldp, eps, momentum, training, (float*)bn_state);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_proj_bn_fwd_dt(const void* y, int32_t dtype, const void* bn_state, const void* wpack,
                                  const float* bias, int32_t B, int32_t Cin, int64_t HW, void* zn, float* inv_norm,
                                  void* stream) {
  PCL_REQUIRE(bn_state && ((uintptr_t)bn_state & 15) == 0 && bn_dtype_ok(dtype) && bn_shape_ok(B, Cin, HW));
  const proj::Layout L = proj::layout(B, Cin, HW);
  const proj::BnPro bn{(const float*)bn_state, y, nullptr, L.ldp};
  if (dtype == PCL_DT_F32)
    return proj_fwd<float, true>((const float*)y, wpack, bias, B, Cin, HW, (float*)zn, inv_norm, stream, bn);
  return proj_fwd<__nv_bfloat16, true>((const __nv_bfloat16*)y, wpack, bias, B, Cin, HW, (__nv_bfloat16*)zn, inv_norm,
                                       stream, bn);
}

extern "C" int pcl_proj_bn_bwd_dt(const void* y, int32_t dtype, const void* bn_state, const void* zn,
                                  const float* inv_norm, const void* gzn, const void* wpack, int32_t B, int32_t Cin,
                                  int64_t HW, void* scratch, void* gu, float* gw, float* gb, float* gsum, float* ggamma,
                                  float* gbeta, void* stream) {
  PCL_REQUIRE(bn_state && ((uintptr_t)bn_state & 15) == 0 && gsum && scratch && bn_dtype_ok(dtype) &&
              bn_shape_ok(B, Cin, HW));
  const proj::Layout L = proj::layout(B, Cin, HW);
  float* part = (float*)((uint8_t*)scratch + L.bn_part_off);
  const proj::BnPro bn{(const float*)bn_state, y, part, L.ldp};
  int st;
  if (dtype == PCL_DT_F32)
    st = proj_bwd<float, true>((const float*)y, (const float*)zn, inv_norm, (const float*)gzn, wpack, B, Cin, HW,
                               scratch, (float*)gu, gw, gb, stream, bn);
  else
    st = proj_bwd<__nv_bfloat16, true>((const __nv_bfloat16*)y, (const __nv_bfloat16*)zn, inv_norm,
                                       (const __nv_bfloat16*)gzn, wpack, B, Cin, HW, scratch, (__nv_bfloat16*)gu, gw,
                                       gb, stream, bn);
  if (st != PCL_OK) return st;
  proj::k_tile_sum<float><<<(unsigned)ceil_div(Cin, 32), proj::TS_NT, 0, (cudaStream_t)stream>>>(
      part, L.ntiles, Cin, L.ldp, gsum, gbeta, ggamma, 0.);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_proj_bn_input_grad_dt(const void* y, int32_t dtype, const void* bn_state, const float* gsum,
                                         int32_t B, int32_t Cin, int64_t HW, int32_t training, void* g, void* stream) {
  PCL_REQUIRE(y && g && bn_state && bn_dtype_ok(dtype) && bn_shape_ok(B, Cin, HW));
  PCL_REQUIRE(training == 0 || (training == 1 && gsum));
  const proj::Layout L = proj::layout(B, Cin, HW);
  const dim3 grid((unsigned)((int64_t)B * Cin), (unsigned)ceil_div64(HW, (int64_t)proj::IG_NT * proj::IG_UNROLL));
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == PCL_DT_F32)
    proj::k_bn_input_grad<float><<<grid, proj::IG_NT, 0, s>>>((const float*)y, (float*)g, (const float*)bn_state, gsum,
                                                              Cin, L.ldp, HW, training);
  else
    proj::k_bn_input_grad<__nv_bfloat16><<<grid, proj::IG_NT, 0, s>>>(
        (const __nv_bfloat16*)y, (__nv_bfloat16*)g, (const float*)bn_state, gsum, Cin, L.ldp, HW, training);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

// (4) the head's first 1x1 convolution (see the kernels above)
extern "C" int64_t pcl_proj_conv1_workspace_bytes(int32_t B, int32_t C, int64_t HW, int32_t which) {
  if (!proj::conv1_shape_ok(B, C, HW) || which < 0 || which > 2) return PCL_ERR_ARG;
  const proj::Conv1Layout L = proj::conv1_layout(B, C, HW);
  return which == 0 ? L.pack_bytes : which == 1 ? L.fwd_bytes : L.bwd_bytes;
}

extern "C" int pcl_proj_conv1_pack(const float* w1, int32_t C, void* pack, void* stream) {
  PCL_REQUIRE(w1 && pack && C > 0 && C <= (1 << 20));
  const proj::Conv1Layout L = proj::conv1_layout(1, C, 1);
  uint8_t* base = (uint8_t*)pack;
  const int64_t n = (int64_t)L.np * L.kp;
  proj::k_pack_bf16<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(
      w1, C, C, L.np, L.kp, L.np, L.kp, (__nv_bfloat16*)base, (__nv_bfloat16*)(base + L.wt_off));
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

// out (B, C, HW) = W a per pixel, W = one of the packed (np, kp) bf16 matrices
template <class T>
static int conv1_gemm(const T* a, const void* wmat, const float* bias, int32_t B, int32_t C, int64_t HW, T* out,
                      double* part, cudaStream_t s) {
  const proj::Conv1Layout L = proj::conv1_layout(B, C, HW);
  CUtensorMap tmW;
  int st = tc_make_tmap(&tmW, wmat, (uint64_t)L.kp, (uint64_t)L.np, proj::DOUT);
  if (st != PCL_OK) return st;
  proj::Conv1Args<T> g{a, bias, out, part, C, L.kp / proj::BK, L.nbands, L.np, HW, L.tiles_per_img};
  const size_t smem = sizeof(proj::FwdSmem) + 1024;
  PCL_SMEM_OPT_IN((proj::k_conv1_gemm<T>), smem);
  proj::k_conv1_gemm<T><<<(unsigned)(L.ptiles * L.nbands), proj::NT, smem, s>>>(tmW, g);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

template <class T>
static int conv1_fwd(const T* x, const void* pack, const float* b1, int32_t B, int32_t C, int64_t HW, T* y,
                     double* sums, void* scratch, cudaStream_t s) {
  const proj::Conv1Layout L = proj::conv1_layout(B, C, HW);
  double* part = sums ? (double*)scratch : nullptr;
  const int st = conv1_gemm(x, pack, b1, B, C, HW, y, part, s);
  if (st != PCL_OK || !sums) return st;
  proj::k_tile_sum<double><<<(unsigned)ceil_div(C, 32), proj::TS_NT, 0, s>>>(part, L.ptiles, C, L.np, sums, nullptr,
                                                                             nullptr, (double)B * (double)HW);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_proj_conv1_fwd_dt(const void* x, int32_t dtype, const void* pack, const float* b1, int32_t B,
                                     int32_t C, int64_t HW, void* y, double* sums, void* scratch, void* stream) {
  PCL_REQUIRE(x && pack && y && (!sums || scratch) && bn_dtype_ok(dtype) && proj::conv1_shape_ok(B, C, HW));
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == PCL_DT_F32) return conv1_fwd((const float*)x, pack, b1, B, C, HW, (float*)y, sums, scratch, s);
  return conv1_fwd((const __nv_bfloat16*)x, pack, b1, B, C, HW, (__nv_bfloat16*)y, sums, scratch, s);
}

template <class T>
static int conv1_bwd(const T* x, const T* gy, const void* pack, int32_t B, int32_t C, int64_t HW, void* scratch,
                     T* gx, float* gw1, float* gb1, cudaStream_t s) {
  const proj::Conv1Layout L = proj::conv1_layout(B, C, HW);
  const proj::Layout& W = L.w;
  uint8_t* sc = (uint8_t*)scratch;
  __nv_bfloat16* gyb = (__nv_bfloat16*)sc;
  float* part = (float*)(sc + L.part_off);
  if (gx) {
    const int st = conv1_gemm(gy, (const uint8_t*)pack + L.wt_off, nullptr, B, C, HW, gx, nullptr, s);
    if (st != PCL_OK) return st;
  }
  const dim3 grid((unsigned)((int64_t)B * L.np), (unsigned)ceil_div64(W.HWp, (int64_t)proj::GP_NT * proj::GP_UNROLL));
  proj::k_conv1_gy_pack<T><<<grid, proj::GP_NT, 0, s>>>(gy, B, C, HW, W.HWp, gyb);
  PCL_LAUNCH_CHECK();
  for (int j = 0; j < L.nbands; ++j) {
    const int n0 = j * proj::DOUT, rows = C - n0 < proj::DOUT ? C - n0 : proj::DOUT;
    const int st = proj_wgrad<T, false>(gyb + (int64_t)n0 * B * W.HWp, x, B, C, HW, W, part, rows,
                                        gw1 + (int64_t)n0 * C, gb1 ? gb1 + n0 : nullptr, proj::BnPro{}, s);
    if (st != PCL_OK) return st;
  }
  return PCL_OK;
}

extern "C" int pcl_proj_conv1_bwd_dt(const void* x, int32_t dtype, const void* gy, const void* pack, int32_t B,
                                     int32_t C, int64_t HW, void* scratch, void* gx, float* gw1, float* gb1,
                                     void* stream) {
  PCL_REQUIRE(x && gy && pack && scratch && gw1 && bn_dtype_ok(dtype) && proj::conv1_shape_ok(B, C, HW));
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == PCL_DT_F32)
    return conv1_bwd((const float*)x, (const float*)gy, pack, B, C, HW, scratch, (float*)gx, gw1, gb1, s);
  return conv1_bwd((const __nv_bfloat16*)x, (const __nv_bfloat16*)gy, pack, B, C, HW, scratch, (__nv_bfloat16*)gx,
                   gw1, gb1, s);
}
