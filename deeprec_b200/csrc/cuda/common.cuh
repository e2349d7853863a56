// Common device helpers for the sm_90a kernel library: PTX wrappers (mbarrier, TMA, system-scope acquire/release for NVLink
// peer signalling), small vector types, error macros.  The warpgroup MMA wrappers are in wgmma.cuh.
#pragma once
#include <cstdlib>
#include <map>
#include <mutex>
#include <thread>
#include <tuple>
#ifdef DR_CUDA_EMU
#include "emu/cuda_emu.h"      // g++ build of the SIMT kernels: every CUDA thread is a host thread (CPU CI, ASAN / TSAN over kernel code)
#else
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <stdio.h>

#include "../common/ev_types.h"

#define DR_CUDA_CHECK(expr)                                                                 \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      fprintf(stderr, "[deeprec_cuda] %s failed at %s:%d: %s\n", #expr, __FILE__, __LINE__, \
              cudaGetErrorString(_e));                                                      \
      return (int)_e;                                                                       \
    }                                                                                       \
  } while (0)

#define DR_LAUNCH_CHECK()                       \
  do {                                          \
    cudaError_t _e = cudaGetLastError();        \
    if (_e != cudaSuccess) {                    \
      fprintf(stderr, "[deeprec_cuda] launch failed at %s:%d: %s\n", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return (int)_e;                           \
    }                                           \
  } while (0)

namespace drc {

inline int& pdl_enabled() { static int v = [] { const char* e = getenv("DEEPREC_PDL"); return (e && e[0] == '0') ? 0 : 1; }(); return v; }

#ifdef DR_CUDA_EMU
#define DR_PDL_LAUNCH(kernel, grid, block, smem, stream, ...) \
  (emu::launch(dim3(grid), dim3(block), (size_t)(smem), stream, [&] { kernel(__VA_ARGS__); }), cudaSuccess)
#else
template <typename... KArgs, typename... Args>
inline cudaError_t dr_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#define DR_PDL_LAUNCH(kernel, grid, block, smem, stream, ...) drc::dr_launch_pdl(kernel, dim3(grid), dim3(block), (size_t)(smem), stream, __VA_ARGS__)
#endif


// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe, fewer in an SM-partitioned context): persistent kernels
// size their grids from it.  Queried once per device.
#ifdef DR_CUDA_EMU
inline int num_sms() { return 2; }   // emulated blocks run one after the other: the grid-stride kernels get small grids (any grid size must be correct)
#else
inline int num_sms() {
  static int n[64] = {};
  int d = 0;
  cudaGetDevice(&d);
  d &= 63;
  if (n[d] == 0) {
    int v = 0;
    n[d] = (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) == cudaSuccess && v > 0) ? v : 132;
  }
  return n[d];
}
#endif

// cudaFuncSetAttribute is per DEVICE: a process that drives several GPUs (serving ProcessorGroup: one replica per GPU in one process)
// must raise the dynamic shared-memory limit on each of them.  One flag per (call site, device).
struct DrPerDeviceOnce {
  bool done[64] = {};
  bool& operator()() { int d = 0; cudaGetDevice(&d); return done[d & 63]; }
};

// Resident-block budget (per SM) of the sparse-path kernels.  They run on a side stream next to the wgmma GEMMs
// (1 CTA/SM, up to ~200 KB smem, 384 threads): capping them leaves thread slots so both streams really overlap.
inline int& sparse_blocks_per_sm() { static int v = 16; return v; }
constexpr int64_t kEmptyKey = INT64_MIN;
constexpr int64_t kTombKey = INT64_MIN + 1;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

#ifdef DR_CUDA_EMU
// the same helpers on host atomics (seq_cst where the device code uses release / acquire at system scope)
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
__device__ __forceinline__ void red_release_sys_add(uint32_t* p, uint32_t v) { __atomic_fetch_add(p, v, __ATOMIC_RELEASE); }
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
__device__ __forceinline__ void pdl_wait() {}
__device__ __forceinline__ void pdl_trigger() {}
__device__ __forceinline__ void pdl_sync() {}
__device__ __forceinline__ void prefetch_l2(const void*) {}
__device__ __forceinline__ int4 ld_nc_v4(const void* p) { int4 r; memcpy(&r, p, 16); return r; }
__device__ __forceinline__ int4 ld_v4_volatile(const void* p) { int4 r; memcpy(&r, p, 16); return r; }
__device__ __forceinline__ void st_na_v4(void* p, const int4& v) { memcpy(p, &v, 16); }
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
  atomicAdd(p, a); atomicAdd(p + 1, b); atomicAdd(p + 2, c); atomicAdd(p + 3, d);
}
#else
// ---- system-scope signalling over NVLink (peer flags live in IPC-mapped memory) ---------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_sys_add(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// streaming 16-byte accesses that do not pollute L1 (peer data is L2-bypassed anyway)
// ---- programmatic dependent launch (PDL) -------------------------------------------------------------------------------
// Kernels on the training-step path are launched with cudaLaunchAttributeProgrammaticStreamSerialization (dr_launch_pdl below):
// the next kernel's CTAs may become resident and run their prologue (barrier init, descriptor prefetch, index
// math) while the previous kernel drains.  griddepcontrol.wait blocks until the predecessor grid has completed and its
// memory is visible, so NOTHING that touches global memory may precede pdl_sync() in such a kernel.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// An early trigger lets the dependent grid's CTAs become resident while the primary still runs, which steals SM slots from
// the primary, so the trigger is left implicit (at grid completion) unless DEEPREC_PDL_EARLY is built in.
#ifdef DEEPREC_PDL_EARLY
__device__ __forceinline__ void pdl_sync() { pdl_wait(); pdl_trigger(); }
#else
__device__ __forceinline__ void pdl_sync() { pdl_wait(); }
#endif

// pull a line into L2 without occupying a register / scoreboard slot (software prefetch for latency-bound streaming kernels)
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ int4 ld_nc_v4(const void* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ int4 ld_v4_volatile(const void* p) {
  int4 r;
  asm volatile("ld.volatile.global.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_na_v4(void* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// vectorised fp32 reduction (sm_90+): one L2 atomic transaction for 4 floats
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- TMA (cp.async.bulk.tensor) -----------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(desc) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(desc), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// L2 prefetch of a tensor-map box: no shared memory, no barrier -- lets a producer run further ahead of the smem ring
__device__ __forceinline__ void tma_prefetch_2d(const void* desc, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(desc), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* desc, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(desc), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

#endif  // DR_CUDA_EMU

// volatile scalar loads of words that other threads update with atomics (probe-then-CAS): plain volatile on the device; relaxed atomic
// loads in the emulation build, which is what they mean -- ThreadSanitizer then reports only the races that are NOT this idiom
#ifdef DR_CUDA_EMU
__device__ __forceinline__ int64_t ld_volatile_i64(const int64_t* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
__device__ __forceinline__ int32_t ld_volatile_i32(const int32_t* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
#else
__device__ __forceinline__ int64_t ld_volatile_i64(const int64_t* p) { return *reinterpret_cast<const volatile int64_t*>(p); }
__device__ __forceinline__ int32_t ld_volatile_i32(const int32_t* p) { return *reinterpret_cast<const volatile int32_t*>(p); }
#endif

// idempotent metadata stores that race BY DESIGN with the volatile reads above (every writer stores the same "dirty" mark; the claim winner publishes
// its list index to readers that accept either value): plain stores on the device, relaxed atomic stores in the emulation build
#ifdef DR_CUDA_EMU
#define DR_ST_RACY(lhs, v) __atomic_store_n(&(lhs), (v), __ATOMIC_RELAXED)
#else
#define DR_ST_RACY(lhs, v) (lhs) = (v)
#endif

// 16-byte / 8-byte volatile loads of a slot's metadata words (same PTX text as before the emulation build existed: the SASS of the hot
// probe kernels is unchanged); on the host: relaxed atomic word loads, so ThreadSanitizer sees them as the benign races they are
#ifdef DR_CUDA_EMU
#define DR_LD_V4_VOLATILE(hi, p)                                                                   \
  do {                                                                                             \
    const int* _q = reinterpret_cast<const int*>(p);                                               \
    (hi).x = __atomic_load_n(_q, __ATOMIC_RELAXED); (hi).y = __atomic_load_n(_q + 1, __ATOMIC_RELAXED); \
    (hi).z = __atomic_load_n(_q + 2, __ATOMIC_RELAXED); (hi).w = __atomic_load_n(_q + 3, __ATOMIC_RELAXED); \
  } while (0)
#define DR_LD_V2_VOLATILE_U32(v, p)                                                                \
  do {                                                                                             \
    const unsigned* _q = reinterpret_cast<const unsigned*>(p);                                     \
    (v).x = __atomic_load_n(_q, __ATOMIC_RELAXED); (v).y = __atomic_load_n(_q + 1, __ATOMIC_RELAXED); \
  } while (0)
#else
#define DR_LD_V4_VOLATILE(hi, p) \
  asm volatile("ld.volatile.global.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"((hi).x), "=r"((hi).y), "=r"((hi).z), "=r"((hi).w) : "l"(p))
#define DR_LD_V2_VOLATILE_U32(v, p) asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"((v).x), "=r"((v).y) : "l"(p) : "memory")
#endif

// ---- deterministic reductions ---------------------------------------------------------------------------------------
// Sums over the batch are never accumulated with floating-point atomics across blocks (their order, and so the rounding, would change
// from run to run): every block writes its partial to a workspace and k_det_colsum adds the partials in block order.
// A workspace belongs to one (device, host thread, call site): the producer kernel and its k_det_colsum are two launches, so callers
// on other host threads (serving sessions, ranks of one process) never share one and cannot interleave on it.  Not keyed by stream:
// a CUDA-graph capture runs on its own stream and must reuse the buffer the eager step before it sized (it grows only outside
// capture).  One host thread must not run the same call site on two streams concurrently.  An old buffer is never freed, since
// kernels still in flight may read it.
inline float* dr_workspace(int slot, size_t nfloat, cudaStream_t s) {
  struct Ws { float* p = nullptr; size_t cap = 0; };
  static std::mutex mu;
  static std::map<std::tuple<int, std::thread::id, int>, Ws> pool;
  std::lock_guard<std::mutex> lk(mu);
  int d = 0;
  cudaGetDevice(&d);
  Ws& w = pool[std::make_tuple(d, std::this_thread::get_id(), slot)];
  if (w.cap >= nfloat) return w.p;
#ifndef DR_CUDA_EMU
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone) return nullptr;
#endif
  const size_t n = nfloat + nfloat / 2;
  float* p = nullptr;
  if (cudaMalloc(&p, n * sizeof(float)) != cudaSuccess) return nullptr;
  w.p = p;
  w.cap = n;
  return p;
}
enum { kWsGemmStats = 0, kWsGemmDw = 1, kWsColstats = 2, kWsHead = 3, kWsBnBwd = 4 };

// dst0[c] += scale * sum_r ws[r * ld + c],  dst1[c] += scale * sum_r ws[r * ld + n + c]   (c < n, rows summed in order; dst1 may be null)
static __global__ void k_det_colsum(const float* __restrict__ ws, int rows, int64_t ld, int n, float* __restrict__ dst0, float* __restrict__ dst1,
                                    float scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  float s0 = 0.f, s1 = 0.f;
  for (int r = 0; r < rows; ++r) {
    s0 += ws[(int64_t)r * ld + c];
    if (dst1) s1 += ws[(int64_t)r * ld + n + c];
  }
  dst0[c] += scale * s0;
  if (dst1) dst1[c] += scale * s1;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace drc
