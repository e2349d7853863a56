// CUDA-on-CPU emulation for the SIMT kernels of this library: the SAME .cu sources compile with g++ (-DDR_CUDA_EMU) and run every CUDA
// thread of a block as a real host thread, so that
//   * CI boxes without a GPU execute the kernels' logic (indexing, barriers, warp collectives, atomics) against the PyTorch oracles, and
//   * AddressSanitizer / ThreadSanitizer see every global- and shared-memory access of a kernel (out-of-bounds rows, missing
//     __syncthreads(), non-atomic read-modify-write) -- the host-side twin of `compute-sanitizer --tool memcheck / racecheck`.
// What is emulated: grid / block indices, static and dynamic shared memory, __syncthreads (threads that already returned count as
// arrived), __syncwarp, shfl / ballot / any / all / match_any / activemask, the atomics, the system-scope acquire / release helpers of
// common.cuh, the handful of runtime calls the host wrappers make (device memory == host memory, streams are synchronous), cub's
// DeviceScan / DeviceSelect / DeviceRadixSort entry points.  What is NOT: wgmma / mma.sync / TMA / mbarrier (those kernels are validated on
// hardware only), timing, memory-model weaknesses (x86 is stronger than the GPU: a pass here does not prove a fence is sufficient).
//
// Blocks of one grid run one after the other (a kernel whose blocks wait on each other would deadlock; none of ours do); kernels of
// different host threads run concurrently, which is how the multi-rank flag protocols are exercised (one host thread per emulated rank).
//
// Reference: the reference tests its GPU kernels only on GPU runners (cibuild/gpu-ut.sh); its CPU CI never executes them.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime_api.h>
#include <vector_types.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <map>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

// the attribute spellings of crt/host_defines.h mean nothing to g++: give them their emulation meaning
#undef __global__
#undef __device__
#undef __host__
#undef __shared__
#undef __constant__
#undef __forceinline__
#undef __launch_bounds__
#undef __align__
#undef __noinline__
#define __global__
#define __device__
#define __host__
#define __shared__ static
#define __constant__ static
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __grid_constant__

namespace emu {

// generation barrier; `expected` may change between rounds (threads that returned from the kernel are dropped)
struct Barrier {
  std::mutex m;
  std::condition_variable cv;
  int live = 0, waiting = 0;
  uint64_t gen = 0;
  void reset(int n) { live = n; waiting = 0; }
  void wait() {
    std::unique_lock<std::mutex> l(m);
    const uint64_t g = gen;
    if (++waiting >= live) { waiting = 0; ++gen; cv.notify_all(); return; }
    cv.wait(l, [&] { return gen != g; });
  }
  void drop() {
    std::unique_lock<std::mutex> l(m);
    --live;
    if (live > 0 && waiting >= live) { waiting = 0; ++gen; cv.notify_all(); }
  }
};

struct Warp {
  std::mutex m;
  std::condition_variable cv;
  uint32_t live = 0;            // lanes still inside the kernel
  // one rendezvous per mask value: disjoint sub-masks of a warp (the match_any groups of a dedup, lanes that skipped a branch and already sit in
  // the next full-mask collective) synchronise independently -- every participant of one collective passes the same mask
  struct Group { int waiting = 0; uint64_t gen = 0; };
  std::map<uint32_t, Group> grp;
  uint64_t slot[32];
  void reset(uint32_t lanes) { live = lanes; grp.clear(); }
  void sync(uint32_t mask) {
    std::unique_lock<std::mutex> l(m);
    if (!(mask & live)) return;
    Group& g = grp[mask];
    const uint64_t gen = g.gen;
    if (++g.waiting >= __builtin_popcount(mask & live)) { g.waiting = 0; ++g.gen; cv.notify_all(); return; }
    cv.wait(l, [&] { return g.gen != gen; });
  }
  void drop(int lane) {
    std::unique_lock<std::mutex> l(m);
    live &= ~(1u << lane);
    // lanes parked in a collective whose mask named this lane are released by the lanes that remain (mask & live shrank)
    bool any = false;
    for (auto& kv : grp)
      if (kv.second.waiting > 0 && kv.second.waiting >= __builtin_popcount(kv.first & live)) { kv.second.waiting = 0; ++kv.second.gen; any = true; }
    if (any) cv.notify_all();
  }
};

struct Block {
  Barrier bar;                      // __syncthreads
  Barrier full;                     // block boundaries of the emulation itself (never dropped)
  std::vector<Warp> warps;
  std::vector<char> dyn;            // dynamic shared memory
  std::mutex sh_mu;                 // static shared memory: one allocation per (declaration, size), living as long as the launch
  std::map<std::pair<int, size_t>, std::unique_ptr<char[]>> sh;
};

struct Ctx {
  uint3 tid{0, 0, 0}, bid{0, 0, 0};
  dim3 bdim{1, 1, 1}, gdim{1, 1, 1};
  Block* blk = nullptr;
  int lin = 0;
};
inline thread_local Ctx ctx;

inline void* shared_var(int id, size_t bytes);
inline void* dyn_smem() { return (void*)(((uintptr_t)ctx.blk->dyn.data() + 127) & ~(uintptr_t)127); }

inline void* shared_var(int id, size_t bytes) {
  Block& b = *ctx.blk;
  std::lock_guard<std::mutex> l(b.sh_mu);
  auto& slot = b.sh[{id, bytes}];
  if (!slot) { slot.reset(new char[bytes + 128]); memset(slot.get(), 0, bytes + 128); }
  return (void*)(((uintptr_t)slot.get() + 127) & ~(uintptr_t)127);
}

inline std::atomic<int64_t>& launch_count() { static std::atomic<int64_t> c{0}; return c; }

template <typename F>
inline void launch(dim3 g, dim3 b, size_t smem, cudaStream_t, F&& body) {
  launch_count().fetch_add(1);
  const int nthreads = (int)(b.x * b.y * b.z);
  const int64_t nblocks = (int64_t)g.x * g.y * g.z;
  if (nthreads <= 0 || nblocks <= 0) return;
  Block blk;
  blk.warps = std::vector<Warp>((nthreads + 31) / 32);
  blk.dyn.resize(smem + 256);
  blk.full.reset(nthreads);
  auto worker = [&](int lin) {
    Ctx& c = ctx;
    c.blk = &blk; c.lin = lin; c.bdim = b; c.gdim = g;
    c.tid.x = lin % b.x; c.tid.y = (lin / b.x) % b.y; c.tid.z = lin / (b.x * b.y);
    for (int64_t blki = 0; blki < nblocks; ++blki) {
      c.bid.x = (unsigned)(blki % g.x); c.bid.y = (unsigned)((blki / g.x) % g.y); c.bid.z = (unsigned)(blki / ((int64_t)g.x * g.y));
      if (lin == 0) {
        blk.bar.reset(nthreads);
        for (size_t w = 0; w < blk.warps.size(); ++w) {
          const int lanes = std::min(32, nthreads - (int)w * 32);
          blk.warps[w].reset(lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1u));
        }
      }
      blk.full.wait();
      body();
      blk.warps[lin >> 5].drop(lin & 31);
      blk.bar.drop();
      blk.full.wait();
    }
    c.blk = nullptr;
  };
  if (nthreads == 1) { worker(0); return; }
  std::vector<std::thread> th;
  th.reserve(nthreads - 1);
  for (int t = 1; t < nthreads; ++t) th.emplace_back(worker, t);
  worker(0);
  for (auto& t : th) t.join();
}

template <typename T>
inline uint64_t to_bits(T v) { static_assert(sizeof(T) <= 8, "shuffle payload"); uint64_t u = 0; memcpy(&u, &v, sizeof(T)); return u; }
template <typename T>
inline T from_bits(uint64_t u) { T v; memcpy(&v, &u, sizeof(T)); return v; }

inline Warp& my_warp() { return ctx.blk->warps[ctx.lin >> 5]; }
inline int my_lane() { return ctx.lin & 31; }

// every lane of `mask` publishes a value, then reads what `pick(lane)` names
template <typename T, typename Pick>
inline T exchange(unsigned mask, T v, Pick pick) {
  Warp& w = my_warp();
  __atomic_store_n(&w.slot[my_lane()], to_bits(v), __ATOMIC_RELAXED);
  w.sync(mask);
  const int src = pick(my_lane());
  const T r = ((mask >> src) & 1u) ? from_bits<T>(__atomic_load_n(&w.slot[src], __ATOMIC_RELAXED)) : v;
  w.sync(mask);
  return r;
}

}  // namespace emu

#define threadIdx (emu::ctx.tid)
#define blockIdx (emu::ctx.bid)
#define blockDim (emu::ctx.bdim)
#define gridDim (emu::ctx.gdim)
#define warpSize 32

inline void __syncthreads() { emu::ctx.blk->bar.wait(); }
inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::my_warp().sync(mask); }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __threadfence_block() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __nanosleep(unsigned) { std::this_thread::yield(); }
inline unsigned __activemask() { return emu::my_warp().live; }

template <typename T>
inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  return emu::exchange(mask, v, [=](int lane) { return (lane & ~(width - 1)) | (src & (width - 1)); });
}
template <typename T>
inline T __shfl_xor_sync(unsigned mask, T v, int x, int width = 32) {
  return emu::exchange(mask, v, [=](int lane) { const int s = lane ^ x; return (s & ~(width - 1)) == (lane & ~(width - 1)) ? s : lane; });
}
template <typename T>
inline T __shfl_down_sync(unsigned mask, T v, unsigned d, int width = 32) {
  return emu::exchange(mask, v, [=](int lane) { const int s = lane + (int)d; return (s & ~(width - 1)) == (lane & ~(width - 1)) ? s : lane; });
}
template <typename T>
inline T __shfl_up_sync(unsigned mask, T v, unsigned d, int width = 32) {
  return emu::exchange(mask, v, [=](int lane) { const int s = lane - (int)d; return s >= (lane & ~(width - 1)) ? s : lane; });
}
inline unsigned __ballot_sync(unsigned mask, int pred) {
  emu::Warp& w = emu::my_warp();
  __atomic_store_n(&w.slot[emu::my_lane()], (uint64_t)(pred != 0), __ATOMIC_RELAXED);
  w.sync(mask);
  unsigned r = 0;
  const unsigned m = mask & w.live;
  for (int l = 0; l < 32; ++l) if (((m >> l) & 1u) && __atomic_load_n(&w.slot[l], __ATOMIC_RELAXED)) r |= 1u << l;
  w.sync(mask);
  return r;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, !pred) == 0; }
template <typename T>
inline unsigned __match_any_sync(unsigned mask, T v) {
  emu::Warp& w = emu::my_warp();
  const uint64_t mine = emu::to_bits(v);
  __atomic_store_n(&w.slot[emu::my_lane()], mine, __ATOMIC_RELAXED);
  w.sync(mask);
  unsigned r = 0;
  const unsigned m = mask & w.live;
  for (int l = 0; l < 32; ++l) if (((m >> l) & 1u) && __atomic_load_n(&w.slot[l], __ATOMIC_RELAXED) == mine) r |= 1u << l;
  w.sync(mask);
  return r;
}

// ---- atomics -----------------------------------------------------------------------------------------------------------------------
template <typename T>
inline T emu_atomic_add_int(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline int atomicAdd(int* p, int v) { return emu_atomic_add_int(p, v); }
inline unsigned atomicAdd(unsigned* p, unsigned v) { return emu_atomic_add_int(p, v); }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return emu_atomic_add_int(p, v); }
inline long long atomicAdd(long long* p, long long v) { return emu_atomic_add_int(p, v); }
template <typename F, typename U>
inline F emu_atomic_add_fp(F* p, F v) {
  U* up = reinterpret_cast<U*>(p);
  U old = __atomic_load_n(up, __ATOMIC_RELAXED);
  for (;;) {
    F f; memcpy(&f, &old, sizeof(F));
    const F nf = f + v; U nu; memcpy(&nu, &nf, sizeof(F));
    if (__atomic_compare_exchange_n(up, &old, nu, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return f;
  }
}
inline float atomicAdd(float* p, float v) { return emu_atomic_add_fp<float, uint32_t>(p, v); }
inline double atomicAdd(double* p, double v) { return emu_atomic_add_fp<double, uint64_t>(p, v); }
template <typename T>
inline T emu_cas(T* p, T cmp, T val) { __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST); return cmp; }
inline int atomicCAS(int* p, int c, int v) { return emu_cas(p, c, v); }
inline unsigned atomicCAS(unsigned* p, unsigned c, unsigned v) { return emu_cas(p, c, v); }
inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long c, unsigned long long v) { return emu_cas(p, c, v); }
inline unsigned short atomicCAS(unsigned short* p, unsigned short c, unsigned short v) { return emu_cas(p, c, v); }
template <typename T>
inline T emu_exch(T* p, T v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
inline int atomicExch(int* p, int v) { return emu_exch(p, v); }
inline unsigned atomicExch(unsigned* p, unsigned v) { return emu_exch(p, v); }
inline unsigned long long atomicExch(unsigned long long* p, unsigned long long v) { return emu_exch(p, v); }
inline float atomicExch(float* p, float v) { uint32_t u; memcpy(&u, &v, 4); u = emu_exch(reinterpret_cast<uint32_t*>(p), u); float r; memcpy(&r, &u, 4); return r; }
template <typename T, typename Op>
inline T emu_rmw(T* p, T v, Op op) {
  T old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (!__atomic_compare_exchange_n(p, &old, op(old, v), true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
#define EMU_RMW(name, expr)                                                                                                  \
  inline int name(int* p, int v) { return emu_rmw(p, v, [](int a, int b) { return expr; }); }                                \
  inline unsigned name(unsigned* p, unsigned v) { return emu_rmw(p, v, [](unsigned a, unsigned b) { return expr; }); }       \
  inline unsigned long long name(unsigned long long* p, unsigned long long v) {                                              \
    return emu_rmw(p, v, [](unsigned long long a, unsigned long long b) { return expr; });                                   \
  }                                                                                                                          \
  inline long long name(long long* p, long long v) { return emu_rmw(p, v, [](long long a, long long b) { return expr; }); }
EMU_RMW(atomicMax, a > b ? a : b)
EMU_RMW(atomicMin, a < b ? a : b)
EMU_RMW(atomicOr, a | b)
EMU_RMW(atomicAnd, a & b)
EMU_RMW(atomicXor, a ^ b)
#undef EMU_RMW
inline unsigned atomicSub(unsigned* p, unsigned v) { return __atomic_fetch_sub(p, v, __ATOMIC_RELAXED); }
inline int atomicSub(int* p, int v) { return __atomic_fetch_sub(p, v, __ATOMIC_RELAXED); }
inline unsigned atomicInc(unsigned* p, unsigned lim) { return emu_rmw(p, lim, [](unsigned a, unsigned l) { return a >= l ? 0u : a + 1u; }); }

// ---- device math / bit intrinsics -------------------------------------------------------------------------------------------------------
inline float __expf(float x) { return expf(x); }
inline float __logf(float x) { return logf(x); }
inline float __fdividef(float a, float b) { return a / b; }
inline float __frcp_rn(float a) { return 1.f / a; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float rsqrtf(float x) { return 1.f / sqrtf(x); }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __saturatef(float x) { return x < 0.f ? 0.f : x > 1.f ? 1.f : x; }
inline int __float2int_rn(float x) { return (int)nearbyintf(x); }
inline int __float2int_rz(float x) { return (int)x; }
inline float __int2float_rn(int x) { return (float)x; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
inline long long __double_as_longlong(double d) { long long u; memcpy(&u, &d, 8); return u; }
inline double __longlong_as_double(long long u) { double d; memcpy(&d, &u, 8); return d; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((x >> i) & 1u) << (31 - i); return r; }
inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
template <typename T>
inline T __ldg(const T* p) { return *p; }
template <typename T>
inline T __ldcs(const T* p) { return *p; }
template <typename T>
inline void __stcs(T* p, T v) { *p = v; }
inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)(uintptr_t)p; }
inline void __trap() { fprintf(stderr, "[cuda_emu] __trap()\n"); abort(); }

// CUDA's integer min / max overload set (mixed widths promote as in device code)
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline long min(long a, long b) { return a < b ? a : b; }
inline long max(long a, long b) { return a > b ? a : b; }
inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }
inline long min(long a, int b) { return a < b ? a : b; }
inline long min(int a, long b) { return a < b ? a : b; }
inline long max(long a, int b) { return a > b ? a : b; }
inline long max(int a, long b) { return a > b ? a : b; }
inline float min(float a, float b) { return fminf(a, b); }
inline float max(float a, float b) { return fmaxf(a, b); }

// ---- the few templated runtime entry points of cuda_runtime.h ----------------------------------------------------------------------------
template <typename T>
inline cudaError_t cudaFuncSetAttribute(T*, cudaFuncAttribute, int) { return cudaSuccess; }
template <typename T>
inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, T, int, size_t) { *n = 1; return cudaSuccess; }

// ---- cub: the device-wide primitives the kernels' host wrappers call (same two-phase temp-storage protocol) --------------------------------
namespace cub {
struct DeviceScan {
  template <typename In, typename Out>
  static cudaError_t ExclusiveSum(void* tmp, size_t& bytes, In in, Out out, int n, cudaStream_t = nullptr) {
    if (!tmp) { bytes = 256; return cudaSuccess; }
    typename std::remove_reference<decltype(out[0])>::type acc = 0;
    for (int i = 0; i < n; ++i) { const auto v = in[i]; out[i] = acc; acc += v; }
    return cudaSuccess;
  }
  template <typename In, typename Out>
  static cudaError_t InclusiveSum(void* tmp, size_t& bytes, In in, Out out, int n, cudaStream_t = nullptr) {
    if (!tmp) { bytes = 256; return cudaSuccess; }
    typename std::remove_reference<decltype(out[0])>::type acc = 0;
    for (int i = 0; i < n; ++i) { acc += in[i]; out[i] = acc; }
    return cudaSuccess;
  }
};
struct DeviceSelect {
  template <typename In, typename Flag, typename Out, typename Num>
  static cudaError_t Flagged(void* tmp, size_t& bytes, In in, Flag flags, Out out, Num num_out, int n, cudaStream_t = nullptr) {
    if (!tmp) { bytes = 256; return cudaSuccess; }
    int k = 0;
    for (int i = 0; i < n; ++i) if (flags[i]) out[k++] = in[i];
    *num_out = k;
    return cudaSuccess;
  }
};
struct DeviceRadixSort {
  template <typename K, typename V>
  static cudaError_t SortPairs(void* tmp, size_t& bytes, const K* kin, K* kout, const V* vin, V* vout, int n, int = 0, int = sizeof(K) * 8, cudaStream_t = nullptr) {
    if (!tmp) { bytes = 256; return cudaSuccess; }
    std::vector<int> idx(n);
    for (int i = 0; i < n; ++i) idx[i] = i;
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return kin[a] < kin[b]; });
    for (int i = 0; i < n; ++i) { kout[i] = kin[idx[i]]; vout[i] = vin[idx[i]]; }
    return cudaSuccess;
  }
};
}  // namespace cub

// ---- runtime calls of the host wrappers: device memory is host memory, streams and events are synchronous ---------------------------------
// (renamed by macro so that an emulation library can live in a process that also has the real libcudart loaded, e.g. next to PyTorch)
namespace emu {
inline cudaError_t rt_malloc(void** p, size_t n) { *p = n ? aligned_alloc(256, (n + 255) / 256 * 256) : nullptr; return (*p || !n) ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t rt_free(void* p) { free(p); return cudaSuccess; }
inline cudaError_t rt_memset(void* p, int v, size_t n) { if (n) memset(p, v, n); return cudaSuccess; }
inline cudaError_t rt_memcpy(void* d, const void* s, size_t n) { if (n) memmove(d, s, n); return cudaSuccess; }
inline cudaError_t rt_ok() { return cudaSuccess; }
}  // namespace emu
template <typename T>
inline cudaError_t emu_cudaMalloc(T** p, size_t n) { return emu::rt_malloc((void**)p, n); }
template <typename T>
inline cudaError_t emu_cudaMallocHost(T** p, size_t n) { return emu::rt_malloc((void**)p, n); }
template <typename T>
inline cudaError_t emu_cudaHostAlloc(T** p, size_t n, unsigned) { return emu::rt_malloc((void**)p, n); }
template <typename T>
inline cudaError_t emu_cudaHostGetDevicePointer(T** d, void* h, unsigned) { *d = (T*)h; return cudaSuccess; }
inline cudaError_t emu_cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { return emu::rt_memcpy(d, s, n); }
inline cudaError_t emu_cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { return emu::rt_memcpy(d, s, n); }
inline cudaError_t emu_cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t = nullptr) { return emu::rt_memset(p, v, n); }
inline cudaError_t emu_cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = nullptr; return cudaSuccess; }
inline cudaError_t emu_cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = nullptr; return cudaSuccess; }
inline cudaError_t emu_cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
inline cudaError_t emu_cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline const char* emu_cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
#define cudaMalloc emu_cudaMalloc
#define cudaMallocHost emu_cudaMallocHost
#define cudaHostAlloc emu_cudaHostAlloc
#define cudaHostGetDevicePointer emu_cudaHostGetDevicePointer
#define cudaFree emu::rt_free
#define cudaFreeHost emu::rt_free
#define cudaMemcpyAsync emu_cudaMemcpyAsync
#define cudaMemcpy emu_cudaMemcpy
#define cudaMemsetAsync emu_cudaMemsetAsync
#define cudaMemset emu::rt_memset
#define cudaStreamSynchronize(s) emu::rt_ok()
#define cudaDeviceSynchronize() emu::rt_ok()
#define cudaGetLastError() emu::rt_ok()
#define cudaPeekAtLastError() emu::rt_ok()
#define cudaSetDevice(d) emu::rt_ok()
#define cudaGetDevice emu_cudaGetDevice
#define cudaGetErrorString emu_cudaGetErrorString
#define cudaStreamCreateWithFlags emu_cudaStreamCreateWithFlags
#define cudaStreamDestroy(s) emu::rt_ok()
#define cudaEventCreateWithFlags emu_cudaEventCreateWithFlags
#define cudaEventRecord emu_cudaEventRecord
#define cudaEventSynchronize(e) emu::rt_ok()
#define cudaEventDestroy(e) emu::rt_ok()
#define cudaStreamWaitEvent(s, e, f) emu::rt_ok()
// CUDA IPC: "another process's allocation" is just the pointer (emulated ranks are threads of one process)
inline cudaError_t emu_cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h, &p, sizeof(p)); return cudaSuccess; }
inline cudaError_t emu_cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, &h, sizeof(*p)); return cudaSuccess; }
inline cudaError_t emu_cudaDeviceCanAccessPeer(int* ok, int, int) { *ok = 1; return cudaSuccess; }
#define cudaIpcGetMemHandle emu_cudaIpcGetMemHandle
#define cudaIpcOpenMemHandle emu_cudaIpcOpenMemHandle
#define cudaIpcCloseMemHandle(p) emu::rt_ok()
#define cudaDeviceCanAccessPeer emu_cudaDeviceCanAccessPeer
