// TEST INFRASTRUCTURE — never part of the product.
//
// Host-side execution model for the engine's SIMT kernels, so that CPU-only test runs (-m "not gpu") execute the REAL
// kernel sources of contrastiveseg_b200/csrc (selection, sampling plan, exact fp32 sweeps, top-k select, bank update,
// normalise, fused seg-CE, graph rank draw) instead of only their host wiring.  tests/emu/build_emu.py rewrites the
// launch syntax and compiles those .cu files with g++ against this header; the wgmma/TMA tensor path compiles against
// the functional model in shim/ptx_sm90.cuh.
//
// Model: one CUDA block = a set of cooperative fibers (ucontext) inside one OS thread; __syncthreads and the warp
// collectives (__shfl*_sync, __ballot_sync, __all_sync, __syncwarp) are scheduling points with CUDA's semantics for
// exited threads; blocks of a grid run one after another; atomics are plain operations.  Floating point is IEEE with
// contraction off, fmaf explicit — results match the GPU to rounding, not bit for bit.
#pragma once
#include <ucontext.h>
#include <sys/mman.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __maxnreg__(...)
#define __shared__ static
#define __align__(n) alignas(n)
#define PCL_EMULATION 1

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint3 { unsigned x, y, z; };
struct float4 { float x, y, z, w; };
struct float2 { float x, y; };
struct int4 { int x, y, z, w; };
struct int2 { int x, y; };
struct uint4 { unsigned x, y, z, w; };
struct uint2 { unsigned x, y; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }

typedef void* cudaStream_t;
enum cudaError_t { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorUnknown = 999 };
typedef cudaError_t cudaError;
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
enum { cudaSharedmemCarveoutMaxShared = 100 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorName(cudaError_t) { return "cudaEmulated"; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated runtime"; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaFree(void*) { return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memmove(d, s, n); return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }

namespace emu {

enum { RUNNABLE = 0, WAIT_BLOCK = 1, WAIT_WARP = 2, DONE = 3, WAIT_NAMED = 4 };
constexpr size_t STACK_BYTES = 256 * 1024;

struct Fiber {
  ucontext_t ctx;
  int state;
  unsigned lin;        // linear thread index in the block
  uint3 t3;
  int named_id = 0, named_n = 0;     // bar.sync id, n (named barrier the fiber waits at)
};
struct Warp { uint64_t buf[32]; };
struct Block {
  std::vector<Fiber> fibers;
  std::vector<Warp> warps;
  ucontext_t sched;
  Fiber* cur = nullptr;
  uint3 bid{0, 0, 0}, bdim{1, 1, 1}, gdim{1, 1, 1};
  void* dyn = nullptr;
  size_t dyn_bytes = 0;
  struct AsyncOp { int engine; std::function<void()> run; };   // engine 0 = TMA (may complete out of order), 1 = in order
  std::deque<AsyncOp> async_q;       // issued-but-not-yet-executed asynchronous operations
  std::function<void()> body;
};
inline Block* g_blk = nullptr;
inline std::vector<void*> g_stacks;

inline void* stack_for(size_t i) {
  while (g_stacks.size() <= i) {
    void* p = mmap(nullptr, STACK_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) { perror("emu: mmap"); abort(); }
    g_stacks.push_back(p);
  }
  return g_stacks[i];
}

inline void yield(int state) {
  Fiber* f = g_blk->cur;
  f->state = state;
  swapcontext(&f->ctx, &g_blk->sched);
}
inline void trampoline() {
  g_blk->body();
  yield(DONE);
}

inline void run_block(Block& B) {
  const size_t n = B.fibers.size();
  for (size_t i = 0; i < n; ++i) {
    Fiber& f = B.fibers[i];
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = stack_for(i);
    f.ctx.uc_stack.ss_size = STACK_BYTES;
    f.ctx.uc_link = nullptr;
    makecontext(&f.ctx, (void (*)())trampoline, 0);
    f.state = RUNNABLE;
  }
  size_t live = n;
  // Scheduling order between synchronisation points is unspecified on the GPU.  PCL_EMU_SCHED=reverse | random[:seed]
  // permutes it (per pass): a result that changes with the order means a missing barrier / a data race.
  static const int sched_mode = [] { const char* e = getenv("PCL_EMU_SCHED"); return !e ? 0 : (e[0] == 'r' && e[1] == 'e') ? 1 : 2; }();
  static uint64_t rng_state = [] { const char* e = getenv("PCL_EMU_SCHED"); const char* c = e ? strchr(e, ':') : nullptr;
                                   return (uint64_t)(c ? atoll(c + 1) : 1) * 0x9E3779B97F4A7C15ull + 1; }();
  std::vector<uint32_t> order(n);
  for (size_t i = 0; i < n; ++i) order[i] = (uint32_t)i;
  while (live) {
    bool progressed = false;
    if (sched_mode == 1) { for (size_t i = 0; i < n; ++i) order[i] = (uint32_t)(n - 1 - i); }
    else if (sched_mode == 2) {
      for (size_t i = n; i > 1; --i) {
        rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
        std::swap(order[i - 1], order[rng_state % i]);
      }
    }
    for (size_t oi = 0; oi < n; ++oi) {
      const size_t i = order[oi];
      Fiber& f = B.fibers[i];
      if (f.state != RUNNABLE) continue;
      B.cur = &f;
      swapcontext(&B.sched, &f.ctx);
      progressed = true;
      if (f.state == DONE) --live;
    }
    // asynchronous engines (TMA / tensor core model): what was issued during this pass executes now, in issue order —
    // i.e. strictly AFTER the issuing thread moved on, so a consumer that does not wait on the mbarrier reads stale data
    // and a producer that refills a stage before its MMAs were committed corrupts their operands (both are caught by
    // the parity checks).  PCL_EMU_ASYNC_DELAY=k executes only every k-th pass (longer in-flight windows).
    if (!B.async_q.empty()) {
      static const int delay = [] { const char* e = getenv("PCL_EMU_ASYNC_DELAY"); int d = e ? atoi(e) : 1; return d < 1 ? 1 : d; }();
      static thread_local unsigned pass_no = 0;
      if (++pass_no % delay == 0 || !progressed) {
        if (sched_mode == 2) {
          // random mode: the tensor pipe retires everything in order; every pending TMA copy completes with probability
          // 1/2, in random order (bulk copies are independent of each other) — at least one operation per drain
          std::deque<Block::AsyncOp> keep;
          std::vector<Block::AsyncOp> tma;
          size_t ran = 0;
          while (!B.async_q.empty()) {
            Block::AsyncOp op = std::move(B.async_q.front()); B.async_q.pop_front();
            if (op.engine == 1) { op.run(); ++ran; } else tma.push_back(std::move(op));
          }
          for (size_t i = tma.size(); i > 1; --i) { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; std::swap(tma[i - 1], tma[rng_state % i]); }
          for (auto& op : tma) {
            rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
            if ((rng_state & 1) || (ran == 0 && !progressed)) { op.run(); ++ran; } else keep.push_back(std::move(op));
          }
          B.async_q = std::move(keep);
        } else {
          while (!B.async_q.empty()) { Block::AsyncOp op = std::move(B.async_q.front()); B.async_q.pop_front(); op.run(); }
        }
        progressed = true;
      }
    }
    // __syncthreads: released when every thread that has not exited waits at it
    bool any = false, all = true;
    for (size_t i = 0; i < n; ++i) {
      const int s = B.fibers[i].state;
      if (s == DONE) continue;
      if (s == WAIT_BLOCK) any = true; else all = false;
    }
    if (any && all) {
      for (size_t i = 0; i < n; ++i) if (B.fibers[i].state == WAIT_BLOCK) B.fibers[i].state = RUNNABLE;
      progressed = true;
    }
    // warp collectives: released per warp when every live lane of the warp waits at one
    for (size_t w = 0; w * 32 < n; ++w) {
      bool wany = false, wall = true;
      for (size_t i = w * 32; i < n && i < w * 32 + 32; ++i) {
        const int s = B.fibers[i].state;
        if (s == DONE) continue;
        if (s == WAIT_WARP) wany = true; else wall = false;
      }
      if (wany && wall) {
        for (size_t i = w * 32; i < n && i < w * 32 + 32; ++i) if (B.fibers[i].state == WAIT_WARP) B.fibers[i].state = RUNNABLE;
        progressed = true;
      }
    }
    // bar.sync id, n: released when n live threads wait at the same id
    for (int id = 1; id < 16; ++id) {
      size_t cnt = 0; int need = 0;
      for (size_t i = 0; i < n; ++i) if (B.fibers[i].state == WAIT_NAMED && B.fibers[i].named_id == id) { ++cnt; need = B.fibers[i].named_n; }
      if (cnt && (int)cnt >= need) {
        for (size_t i = 0; i < n; ++i) if (B.fibers[i].state == WAIT_NAMED && B.fibers[i].named_id == id) B.fibers[i].state = RUNNABLE;
        progressed = true;
      }
    }
    if (!progressed) { fprintf(stderr, "emu: deadlock (divergent barrier) in block (%u,%u,%u)\n", B.bid.x, B.bid.y, B.bid.z); abort(); }
  }
}

struct Cfg { dim3 g, b; size_t smem; };
inline Cfg cfg_make(dim3 g, dim3 b, size_t smem = 0, cudaStream_t = nullptr) { return Cfg{g, b, smem}; }

inline void launch(const Cfg& c, std::function<void()> body) {
  Block B;
  const unsigned nt = c.b.x * c.b.y * c.b.z;
  if (nt == 0 || nt > 1024) { fprintf(stderr, "emu: bad block size %u\n", nt); abort(); }
  B.fibers.resize(nt);
  B.warps.resize((nt + 31) / 32);
  B.bdim = uint3{c.b.x, c.b.y, c.b.z};
  B.gdim = uint3{c.g.x, c.g.y, c.g.z};
  B.body = std::move(body);
  std::vector<char> dyn(c.smem + 2048);
  B.dyn = (void*)(((uintptr_t)dyn.data() + 1023) & ~(uintptr_t)1023);      // 1024-aligned like the shared window
  B.dyn_bytes = c.smem + 1024;
  for (unsigned i = 0; i < nt; ++i) {
    B.fibers[i].lin = i;
    B.fibers[i].t3 = uint3{i % c.b.x, (i / c.b.x) % c.b.y, i / (c.b.x * c.b.y)};
  }
  Block* saved = g_blk;
  g_blk = &B;
  // blocks of a grid run one after another; with PCL_EMU_SCHED set their order is reversed / shuffled as well (no kernel
  // may depend on the order in which its blocks are scheduled)
  const size_t nb = (size_t)c.g.x * c.g.y * c.g.z;
  std::vector<size_t> border(nb);
  for (size_t i = 0; i < nb; ++i) border[i] = i;
  const char* sched = getenv("PCL_EMU_SCHED");
  if (sched && sched[0] == 'r' && sched[1] == 'e') { for (size_t i = 0; i < nb; ++i) border[i] = nb - 1 - i; }
  else if (sched) {
    uint64_t st = 0x9E3779B97F4A7C15ull * (nb + 1) + (uint64_t)c.b.x;
    for (size_t i = nb; i > 1; --i) { st ^= st << 13; st ^= st >> 7; st ^= st << 17; std::swap(border[i - 1], border[st % i]); }
  }
  for (size_t bi = 0; bi < nb; ++bi) {
    const size_t lin = border[bi];
    B.bid = uint3{(unsigned)(lin % c.g.x), (unsigned)((lin / c.g.x) % c.g.y), (unsigned)(lin / ((size_t)c.g.x * c.g.y))};
    run_block(B);
  }
  g_blk = saved;
}

template <class... P>
struct Bound {
  void (*k)(P...);
  Cfg c;
  template <class... A>
  void operator()(A&&... a) const {
    void (*kk)(P...) = k;
    launch(c, [&]() { kk(static_cast<P>(a)...); });
  }
};
struct CfgBinder {
  Cfg c;
  template <class... P> Bound<P...> bind(void (*k)(P...)) const { return Bound<P...>{k, c}; }
};
template <class G, class Bk>
inline CfgBinder cfg(G g, Bk b, size_t smem = 0, cudaStream_t s = nullptr) { return CfgBinder{cfg_make(dim3(g), dim3(b), smem, s)}; }

inline void* dyn_smem() { return g_blk->dyn; }
// Fixed-size 1-D __shared__ arrays (build_emu.py rewrites `__shared__ T a[N];` to `__shared__ SharedArray<T, N> a;`):
// an index outside [0, N) aborts, as the access would fault or corrupt a neighbouring array on the GPU.  On the host
// the array is a process static, and a write past it lands in neighbouring storage that nothing reads back wrong, so
// the overflow would go unseen.  Decays to T* like the array it stands for; pointer arithmetic is not checked.
template <class T, long long N>
struct SharedArray {
  T v[N];
  template <class I> T& operator[](I i) {
    if ((long long)i < 0 || (long long)i >= N) {
      fprintf(stderr, "emu: __shared__ array index %lld outside [0, %lld)\n", (long long)i, N);
      abort();
    }
    return v[i];
  }
  operator T*() { return v; }
};
inline void named_barrier(int id, int nthreads) {
  Fiber* f = g_blk->cur;
  f->named_id = id; f->named_n = nthreads;
  yield(WAIT_NAMED);
}
// cooperative spin (polling loops on mbarriers): stay runnable, let the other fibers of the block run
inline void spin_yield() { yield(RUNNABLE); }
inline unsigned lane_id() { return g_blk->cur->lin & 31u; }
inline Warp& my_warp() { return g_blk->warps[g_blk->cur->lin >> 5]; }
inline bool lane_live(unsigned lane) {
  const size_t i = (size_t)(g_blk->cur->lin & ~31u) + lane;
  return i < g_blk->fibers.size() && g_blk->fibers[i].state != DONE;
}

template <class T> inline uint64_t to_bits(T v) { uint64_t b = 0; static_assert(sizeof(T) <= 8, "shuffle width"); memcpy(&b, &v, sizeof(T)); return b; }
template <class T> inline T from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }

template <class T> inline T shfl_from(T v, unsigned src, bool use_src) {
  Warp& W = my_warp();
  W.buf[lane_id()] = to_bits(v);
  yield(WAIT_WARP);
  T r = use_src ? from_bits<T>(W.buf[src & 31u]) : v;
  yield(WAIT_WARP);
  return r;
}

}  // namespace emu

#define threadIdx (emu::g_blk->cur->t3)
#define blockIdx (emu::g_blk->bid)
#define blockDim (emu::g_blk->bdim)
#define gridDim (emu::g_blk->gdim)

static inline void __syncthreads() { emu::yield(emu::WAIT_BLOCK); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::yield(emu::WAIT_WARP); }
template <class T> static inline T __shfl_sync(unsigned, T v, int src) { return emu::shfl_from(v, (unsigned)src, true); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m) { return emu::shfl_from(v, emu::lane_id() ^ (unsigned)m, true); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d) {
  const unsigned l = emu::lane_id();
  return emu::shfl_from(v, l - d, l >= d);
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d) {
  const unsigned l = emu::lane_id();
  return emu::shfl_from(v, l + d, l + d < 32);
}
static inline unsigned __ballot_sync(unsigned, int pred) {
  emu::Warp& W = emu::my_warp();
  W.buf[emu::lane_id()] = pred ? 1u : 0u;
  emu::yield(emu::WAIT_WARP);
  unsigned m = 0;
  for (unsigned l = 0; l < 32; ++l) if (emu::lane_live(l) && W.buf[l]) m |= 1u << l;
  emu::yield(emu::WAIT_WARP);
  return m;
}
static inline int __all_sync(unsigned, int pred) {
  emu::Warp& W = emu::my_warp();
  W.buf[emu::lane_id()] = pred ? 1u : 0u;
  emu::yield(emu::WAIT_WARP);
  int all = 1;
  for (unsigned l = 0; l < 32; ++l) if (emu::lane_live(l) && !W.buf[l]) all = 0;
  emu::yield(emu::WAIT_WARP);
  return all;
}
static inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0; }

template <class T, class U> static inline T atomicAdd(T* p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicMax(T* p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMin(T* p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicOr(T* p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> static inline T atomicExch(T* p, U v) { T o = *p; *p = (T)v; return o; }

static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
#define __expf(x) expf(x)      /* glibc declares __expf / __logf itself */
#define __logf(x) logf(x)
static inline float __fdividef(float a, float b) { return a / b; }
static inline long long __float2ll_rn(float x) { return llrintf(x); }
static inline int __float2int_rn(float x) { return (int)lrintf(x); }
static inline void __trap() { fprintf(stderr, "emu: __trap()\n"); abort(); }
#define __grid_constant__
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
// a small "GPU" keeps persistent grids short under emulation and still exercises multi-CTA work splitting; builds with
// -DPCL_EMU_SMS=n model an n-SM part (132: H100 SXM, 114: H100 PCIe) to reach the work splits of a real device
#ifndef PCL_EMU_SMS
#define PCL_EMU_SMS 6
#endif
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = PCL_EMU_SMS; return cudaSuccess; }
enum cudaDriverEntryPointQueryResult { cudaDriverEntryPointSuccess = 0, cudaDriverEntryPointSymbolNotFound = 1 };
enum { cudaEnableDefault = 0 };
cudaError_t cudaGetDriverEntryPoint(const char* symbol, void** fn, unsigned long long flags, cudaDriverEntryPointQueryResult* q);
static inline int __clz(int x) { return x == 0 ? 32 : __builtin_clz((unsigned)x); }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline void __threadfence() {}
static inline unsigned int __umulhi(unsigned int a, unsigned int b) { return (unsigned int)(((unsigned long long)a * b) >> 32); }
static inline void __nanosleep(unsigned) {}
template <class A, class B> static inline auto min(A a, B b) -> decltype(a + b) { return a < b ? a : b; }
template <class A, class B> static inline auto max(A a, B b) -> decltype(a + b) { return a > b ? a : b; }
