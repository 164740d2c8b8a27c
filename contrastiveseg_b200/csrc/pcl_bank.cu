// Memory-bank kernels (SURVEY §8 rows a7, a8) — replace segmentor/trainer_contrastive.py:102-138.
//
// The reference loops in Python over (image, class) with unique/nonzero/mean/randperm/normalize and an
// int(ptr) host sync per pair.  Here:
//   k_bank_counts   per-image pixel count of every class in the sub-sampled label grid (labels[:, ::s, ::s])
//   k_bank_segsum   segment sums of the key features per (image, class): ONE pass over the keys, integer
//                   (fixed-point, 2^-36) accumulation so the result does not depend on atomic ordering
//   k_bank_rows     the enqueue packet: normalised segment mean + K' normalised pixel rows per slot
//   k_bank_apply    ordered application of the packets of all ranks (ring-buffer quirks Q2, Q4; overlap
//                   between successive writes resolved in (rank, image) order exactly like the Python loop),
//                   also refreshes the bf16 class-blocked shadow rows
// HBM traffic per call: keys read once (<= B*D*h*w*4 B) + labels grid + ~B*(K-1)*(1+F)*D*4 B of rows.
#include "pcl_common.cuh"

namespace pcl {

constexpr float FIX_SCALE = 68719476736.f;          // 2^36
constexpr double FIX_INV = 1.0 / 68719476736.0;
constexpr int SEG_DG = 8;                            // channels per CTA in k_bank_segsum
constexpr int SEG_PX = 2048;                         // grid positions per CTA

struct BankDims {
  pcl_bank_geom g;
  int Hs, Ws, T;        // sub-sampled label grid, T = Hs*Ws positions (== feature columns, Q6)
  int64_t HW;
  int slot_f32;
};

__device__ __forceinline__ int grid_label(const BankDims& d, const int64_t* __restrict__ lab_b, int t) {
  int gy = t / d.Ws, gx = t - gy * d.Ws;
  int64_t v = lab_b[(int64_t)gy * d.g.network_stride * d.g.Wimg + (int64_t)gx * d.g.network_stride];
  return (v > 0 && v < d.g.K) ? (int)v : -1;        // class 0 and ignore never enter the bank (Q2)
}

__global__ void __launch_bounds__(256)
k_bank_counts(BankDims d, const int64_t* __restrict__ labels, int32_t* __restrict__ counts) {
  extern __shared__ int s_cnt[];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < d.g.K; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  const int64_t* lab_b = labels + (int64_t)b * d.g.Himg * d.g.Wimg;
  for (int t = blockIdx.x * SEG_PX + threadIdx.x; t < min(d.T, (int)(blockIdx.x + 1) * SEG_PX); t += blockDim.x) {
    int c = grid_label(d, lab_b, t);
    if (c > 0) atomicAdd(&s_cnt[c], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d.g.K; i += blockDim.x)
    if (s_cnt[i]) atomicAdd(&counts[b * d.g.K + i], s_cnt[i]);
}

template <typename T>       // element type of keys (converted on load: the sums equal those of the fp32 copy)
__global__ void __launch_bounds__(256)
k_bank_segsum(BankDims d, const T* __restrict__ keys, const int64_t* __restrict__ labels,
              unsigned long long* __restrict__ sums) {
  extern __shared__ unsigned long long s_bins[];      // [K][SEG_DG]
  const int b = blockIdx.z, d0 = blockIdx.y * SEG_DG, t0 = blockIdx.x * SEG_PX;
  const int K = d.g.K, D = d.g.D;
  for (int i = threadIdx.x; i < K * SEG_DG; i += blockDim.x) s_bins[i] = 0ull;
  __syncthreads();
  const int64_t* lab_b = labels + (int64_t)b * d.g.Himg * d.g.Wimg;
  constexpr int PER = SEG_PX / 256;
  int cls[PER];
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    int t = t0 + u * 256 + threadIdx.x;
    cls[u] = t < d.T ? grid_label(d, lab_b, t) : -1;
  }
  const T* kb = keys + (int64_t)b * D * d.HW;
  // Label maps are blocky: most warps see a single class.  Accumulate the thread's own pixels in a register while
  // the class does not change, then reduce class-uniform warps with shuffles -> one shared-memory atomic per warp
  // instead of one per pixel (the per-pixel version serialised on a handful of hot bins: 145 us for one image).
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int dl = 0; dl < SEG_DG; ++dl) {
    if (d0 + dl >= D) break;
    const T* row = kb + (int64_t)(d0 + dl) * d.HW;
    long long acc = 0;
    int acc_cls = -1;
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      if (cls[u] > 0) {
        const long long q = __float2ll_rn(to_f32(row[t0 + u * 256 + threadIdx.x]) * FIX_SCALE);
        if (cls[u] != acc_cls) {
          if (acc_cls > 0) atomicAdd(&s_bins[acc_cls * SEG_DG + dl], (unsigned long long)acc);
          acc = 0;
          acc_cls = cls[u];
        }
        acc += q;
      }
    }
    // warp-level: all lanes hold the same (possibly empty) class -> shuffle reduction, one atomic
    const int c0 = __shfl_sync(0xffffffffu, acc_cls, 0);
    if (__all_sync(0xffffffffu, acc_cls == c0)) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0 && c0 > 0) atomicAdd(&s_bins[c0 * SEG_DG + dl], (unsigned long long)acc);
    } else if (acc_cls > 0) {
      atomicAdd(&s_bins[acc_cls * SEG_DG + dl], (unsigned long long)acc);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * SEG_DG; i += blockDim.x) {
    unsigned long long v = s_bins[i];
    int c = i / SEG_DG, dl = i - c * SEG_DG;
    if (v != 0ull && d0 + dl < D) atomicAdd(&sums[((int64_t)b * K + c) * D + d0 + dl], v);
  }
}

// one CTA per (image, class) slot
template <typename T>
__global__ void __launch_bounds__(256)
k_bank_rows(BankDims d, const T* __restrict__ keys, const int32_t* __restrict__ counts,
            const unsigned long long* __restrict__ sums, const int32_t* __restrict__ ranks, uint64_t seed,
            const unsigned long long* __restrict__ seed_offset, float* __restrict__ packet) {
  if (seed_offset != nullptr) seed += *seed_offset;          // captured sequence: per-replay part lives on the device
  const int slot = blockIdx.x;
  const int K = d.g.K, D = d.g.D, F = d.g.pixel_update_freq;
  const int b = slot / K, c = slot - b * K;
  float* out = packet + (int64_t)slot * d.slot_f32;
  const int n = c > 0 ? counts[slot] : 0;
  const int kp = n < F ? n : F;
  if (threadIdx.x == 0) { out[0] = (float)n; out[1] = (float)kp; }
  if (n == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const T* kb = keys + (int64_t)b * D * d.HW;
  for (int row = warp - 1 + 0; row < kp; row += nwarp) {
    // row == -1: segment mean; row >= 0: pixel row
    if (row < 0) {
      const unsigned long long* sm = sums + (int64_t)slot * D;
      float ss = 0.f;
      for (int dd = lane; dd < D; dd += 32) {
        float m = (float)((double)(long long)sm[dd] * FIX_INV / (double)n);
        ss += m * m;
      }
      ss = warp_sum(ss);
      const float den = fmaxf(sqrtf(ss), 1e-12f);          // F.normalize: x / max(||x||, eps)
      for (int dd = lane; dd < D; dd += 32) {
        float m = (float)((double)(long long)sm[dd] * FIX_INV / (double)n);
        out[2 + dd] = m / den;
      }
    } else {
      int col;
      if (ranks != nullptr) col = ranks[(int64_t)slot * F + row];
      else col = (int)keyed_perm((uint32_t)row, (uint32_t)n, mix64(seed ^ (0xB5ull << 56) ^ (uint64_t)slot));
      col = col < 0 ? 0 : (col >= n ? n - 1 : col);           // perm value used directly as the column (Q5)
      float ss = 0.f;
      for (int dd = lane; dd < D; dd += 32) {
        float v = to_f32(kb[(int64_t)dd * d.HW + col]);
        ss += v * v;
      }
      ss = warp_sum(ss);
      const float den = fmaxf(sqrtf(ss), 1e-12f);
      float* o = out + 2 + D + (int64_t)row * D;
      for (int dd = lane; dd < D; dd += 32) o[dd] = to_f32(kb[(int64_t)dd * d.HW + col]) / den;
    }
  }
}

// one CTA per class.  The reference applies the (rank, image) slots of a class one after another (ring-buffer quirks Q2,
// Q4: the pixel pointer advances by ONE per slot, so successive windows overlap and a later slot overwrites rows of an
// earlier one).  Nothing reads the bank during the apply, so the result only depends on WHO WRITES LAST: thread 0 replays
// the pointer arithmetic of all slots (integers only), then every row is copied once, in parallel, by its last writer.
// (A sequential apply costs one dependent chain per packet, which grows with the number of ranks.)
constexpr int APPLY_MAX_SLOTS = 1024;            // world * B slots of one class handled in shared memory

__global__ void __launch_bounds__(256)
k_bank_apply(BankDims d, const float* __restrict__ packets, int world, int64_t packet_f32, float* __restrict__ segq,
             int64_t* __restrict__ seg_ptr, float* __restrict__ pixq, int64_t* __restrict__ pix_ptr,
             __nv_bfloat16* __restrict__ shadow, unsigned long long* enqueue_counter) {
  __shared__ int s_src[APPLY_MAX_SLOTS];         // valid slots in application order: r * B + b
  __shared__ int s_seg[APPLY_MAX_SLOTS];         // segment row written by the slot
  __shared__ int s_dst[APPLY_MAX_SLOTS];         // first pixel row written by the slot
  __shared__ short s_kp[APPLY_MAX_SLOTS];        // number of pixel rows of the slot
  __shared__ int s_n;
  const int c = blockIdx.x;
  // captured sequences: the packet of this step was seeded from *enqueue_counter (pcl_bank_packet_dev); the apply is the
  // last kernel of the step's enqueue, so it advances the counter
  if (c == 0 && threadIdx.x == 0 && enqueue_counter != nullptr) *enqueue_counter += 1ull;
  if (c == 0) return;
  const int K = d.g.K, D = d.g.D, M = d.g.M, B = d.g.B;
  if (threadIdx.x == 0) {
    int sp = (int)seg_ptr[c], pp = (int)pix_ptr[c];
    sp = ((sp % M) + M) % M; pp = ((pp % M) + M) % M;
    int n = 0;
    for (int r = 0; r < world; ++r) {
      for (int b = 0; b < B; ++b) {
        const float* in = packets + (int64_t)r * packet_f32 + (int64_t)(b * K + c) * d.slot_f32;
        const int cnt = (int)in[0];
        if (cnt <= 0) continue;
        const int kp = (int)in[1];
        if (n < APPLY_MAX_SLOTS) {
          s_src[n] = r * B + b;
          s_seg[n] = sp;                                     // trainer_contrastive.py:120-123
          // pixel rows (trainer_contrastive.py:133-138, Q4)
          if (pp + kp >= M) { s_dst[n] = M - kp; pp = 0; }
          else              { s_dst[n] = pp;     pp = (pp + 1) % M; }
          s_kp[n] = (short)kp;
          sp = (sp + 1) % M;
          ++n;
        }
      }
    }
    s_n = n;
    if (n > 0) { seg_ptr[c] = sp; pix_ptr[c] = pp; }
  }
  __syncthreads();
  const int n = s_n;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  // work items: (slot i, row j) with j = -1 the segment row, j in [0, kp) a pixel row; one warp per item
  int item = warp;
  for (int i = 0; i < n; ++i) {
    const int kp = s_kp[i];
    const int src = s_src[i];
    const float* in = packets + (int64_t)(src / B) * packet_f32 + (int64_t)((src % B) * K + c) * d.slot_f32;
    for (int j = -1; j < kp; ++j, --item) {
      if (item != 0) { if (item < 0) item += nwarp; continue; }
      item = nwarp;                                           // next item of this warp
      // is this row overwritten by a later slot?
      bool dead = false;
      if (j < 0) {
        for (int t = i + 1; t < n && !dead; ++t) dead = s_seg[t] == s_seg[i];
        if (!dead) {
          float* srow = segq + ((int64_t)c * M + s_seg[i]) * D;
          for (int dd = lane; dd < D; dd += 32) {
            const float v = in[2 + dd];
            srow[dd] = v;
            if (shadow) shadow[((int64_t)(c - 1) * 2 * M + s_seg[i]) * D + dd] = __float2bfloat16(v);
          }
        }
      } else {
        const int q = s_dst[i] + j;
        for (int t = i + 1; t < n && !dead; ++t) dead = q >= s_dst[t] && q < s_dst[t] + s_kp[t];
        if (!dead) {
          float* prow = pixq + ((int64_t)c * M + q) * D;
          const float* irow = in + 2 + D + (int64_t)j * D;
          for (int dd = lane; dd < D; dd += 32) {
            const float v = irow[dd];
            prow[dd] = v;
            if (shadow) shadow[((int64_t)(c - 1) * 2 * M + M + q) * D + dd] = __float2bfloat16(v);
          }
        }
      }
    }
  }
}

__global__ void k_shadow_rebuild(const float* __restrict__ segq, const float* __restrict__ pixq, int K, int M, int D,
                                 int64_t rows_pad, __nv_bfloat16* __restrict__ shadow) {
  const int64_t total = rows_pad * D;
  const int64_t real = (int64_t)(K - 1) * 2 * M * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < real) {
      int64_t row = i / D;
      int dd = (int)(i - row * D);
      int c = (int)(row / (2 * M)) + 1;
      int q = (int)(row - (int64_t)(c - 1) * 2 * M);
      v = q < M ? segq[((int64_t)c * M + q) * D + dd] : pixq[((int64_t)c * M + (q - M)) * D + dd];
    }
    shadow[i] = __float2bfloat16(v);
  }
}

}  // namespace pcl

using namespace pcl;

static int make_dims(const pcl_bank_geom* g, BankDims* d) {
  if (!g) return PCL_ERR_ARG;
  if (g->B <= 0 || g->D <= 0 || g->h <= 0 || g->w <= 0 || g->Himg <= 0 || g->Wimg <= 0) return PCL_ERR_ARG;
  if (g->K <= 0 || g->K > PCL_MAX_CLASSES || g->M <= 0 || g->network_stride <= 0 || g->pixel_update_freq < 0)
    return PCL_ERR_ARG;
  d->g = *g;
  d->Hs = ceil_div(g->Himg, g->network_stride);
  d->Ws = ceil_div(g->Wimg, g->network_stride);
  d->T = d->Hs * d->Ws;
  d->HW = (int64_t)g->h * g->w;
  d->slot_f32 = 2 + g->D + g->pixel_update_freq * g->D;
  if ((int64_t)d->T > d->HW) return PCL_ERR_SHAPE;     // the reference would index past the feature map
  // K' = min(n, pixel_update_freq) rows go into a ring of M rows: with K' > M the reference's slice assignment
  // pixel_queue[lb, -K':, :] = feat raises (trainer_contrastive.py:133-135).  That needs n > M and freq > M; the engine
  // refuses the configuration up front instead of depending on the data (the wrap branch would write before row 0).
  if (g->pixel_update_freq > g->M) return PCL_ERR_SHAPE;
  return PCL_OK;
}

extern "C" int64_t pcl_bank_packet_floats(const pcl_bank_geom* g) {
  BankDims d;
  int st = make_dims(g, &d);
  if (st != PCL_OK && st != PCL_ERR_SHAPE) return st;
  return (int64_t)g->B * g->K * d.slot_f32;
}

extern "C" int64_t pcl_bank_scratch_floats(const pcl_bank_geom* g) {
  BankDims d;
  int st = make_dims(g, &d);
  if (st != PCL_OK && st != PCL_ERR_SHAPE) return st;
  // counts (int32) + sums (uint64), expressed in floats
  return (int64_t)g->B * g->K + 2 * (int64_t)g->B * g->K * g->D + 2;
}

static int bank_packet_impl(const pcl_bank_geom* g, const void* keys, int keys_dtype, const int64_t* labels,
                            const int32_t* ranks, uint64_t seed, const uint64_t* seed_offset, float* scratch, float* packet,
                            void* stream) {
  BankDims d;
  int st = make_dims(g, &d);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(keys && labels && scratch && packet && dtype_ok(keys_dtype));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t slots = (int64_t)g->B * g->K;
  int32_t* counts = reinterpret_cast<int32_t*>(scratch);
  // 8-byte aligned start for the 64-bit sums
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(scratch + ((slots + 1) / 2) * 2);
  PCL_CUDA(cudaMemsetAsync(scratch, 0, (size_t)(((slots + 1) / 2) * 2 + 2 * slots * g->D) * sizeof(float), s));
  const int chunks = ceil_div(d.T, SEG_PX);
  k_bank_counts<<<dim3(chunks, g->B), 256, g->K * sizeof(int), s>>>(d, labels, counts);
  PCL_LAUNCH_CHECK();
  PCL_DT_SWITCH(keys_dtype, T,
    k_bank_segsum<T><<<dim3(chunks, ceil_div(g->D, SEG_DG), g->B), 256, (size_t)g->K * SEG_DG * sizeof(unsigned long long),
                       s>>>(d, (const T*)keys, labels, sums);)
  PCL_LAUNCH_CHECK();
  PCL_DT_SWITCH(keys_dtype, T,
    k_bank_rows<T><<<(unsigned)slots, 256, 0, s>>>(d, (const T*)keys, counts, sums, ranks, seed,
                                                   reinterpret_cast<const unsigned long long*>(seed_offset), packet);)
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_bank_packet(const pcl_bank_geom* g, const float* keys, const int64_t* labels, const int32_t* ranks,
                               uint64_t seed, float* scratch, float* packet, void* stream) {
  return bank_packet_impl(g, keys, PCL_DT_F32, labels, ranks, seed, nullptr, scratch, packet, stream);
}

extern "C" int pcl_bank_packet_dev(const pcl_bank_geom* g, const float* keys, const int64_t* labels, uint64_t seed,
                                   const uint64_t* seed_offset, float* scratch, float* packet, void* stream) {
  return bank_packet_impl(g, keys, PCL_DT_F32, labels, nullptr, seed, seed_offset, scratch, packet, stream);
}

extern "C" int pcl_bank_packet_dt(const pcl_bank_geom* g, const void* keys, int32_t keys_dtype, const int64_t* labels,
                                  const int32_t* ranks, uint64_t seed, float* scratch, float* packet, void* stream) {
  return bank_packet_impl(g, keys, keys_dtype, labels, ranks, seed, nullptr, scratch, packet, stream);
}

extern "C" int pcl_bank_packet_dev_dt(const pcl_bank_geom* g, const void* keys, int32_t keys_dtype, const int64_t* labels,
                                      uint64_t seed, const uint64_t* seed_offset, float* scratch, float* packet,
                                      void* stream) {
  return bank_packet_impl(g, keys, keys_dtype, labels, nullptr, seed, seed_offset, scratch, packet, stream);
}

extern "C" int pcl_bank_apply(const pcl_bank_geom* g, const float* packets, int32_t world, float* segment_queue,
                              int64_t* segment_queue_ptr, float* pixel_queue, int64_t* pixel_queue_ptr,
                              void* shadow_bf16, void* stream) {
  return pcl_bank_apply_ctr(g, packets, world, segment_queue, segment_queue_ptr, pixel_queue, pixel_queue_ptr, shadow_bf16,
                            nullptr, stream);
}

extern "C" int pcl_bank_apply_ctr(const pcl_bank_geom* g, const float* packets, int32_t world, float* segment_queue,
                                  int64_t* segment_queue_ptr, float* pixel_queue, int64_t* pixel_queue_ptr,
                                  void* shadow_bf16, uint64_t* enqueue_counter, void* stream) {
  BankDims d;
  int st = make_dims(g, &d);
  if (st != PCL_OK) return st;
  PCL_REQUIRE(packets && world >= 1 && segment_queue && segment_queue_ptr && pixel_queue && pixel_queue_ptr);
  // the slots of one class (world * B of them) are replayed in shared memory
  if ((int64_t)world * g->B > APPLY_MAX_SLOTS) return PCL_ERR_UNSUPPORTED;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t packet_f32 = (int64_t)g->B * g->K * d.slot_f32;
  k_bank_apply<<<g->K, 256, 0, s>>>(d, packets, world, packet_f32, segment_queue, segment_queue_ptr, pixel_queue,
                                   pixel_queue_ptr, (__nv_bfloat16*)shadow_bf16,
                                   reinterpret_cast<unsigned long long*>(enqueue_counter));
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}

extern "C" int pcl_bank_shadow_rebuild(const float* segment_queue, const float* pixel_queue, int32_t K, int32_t M,
                                       int32_t D, void* shadow_bf16, void* stream) {
  PCL_REQUIRE(segment_queue && pixel_queue && shadow_bf16 && K >= 1 && M >= 1 && D >= 1);
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t rows = (int64_t)(K - 1) * 2 * M;
  const int64_t rows_pad = ceil_div64(rows > 0 ? rows : 1, 256) * 256;
  k_shadow_rebuild<<<num_sms() * 8, 256, 0, s>>>(segment_queue, pixel_queue, K, M, D, rows_pad, (__nv_bfloat16*)shadow_bf16);
  PCL_LAUNCH_CHECK();
  return PCL_OK;
}
