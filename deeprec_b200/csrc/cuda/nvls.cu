// NVLS (NVLink SHARP) dense all-reduce fused with the optimizer: VMM symmetric allocation + multicast object + multimem.ld_reduce.
//
// Replaces Horovod's ncclAllReduce + separate Apply* op (python/distribute/hvd_strategy.py:391-398, SURVEY §2.15 C1 / K9) for dense nets
// where the one-shot peer pull of k_allreduce_apply (every rank loads all W copies: O(W * P) bytes per rank) stops scaling: with a
// multicast mapping ONE multimem.ld_reduce.add returns the sum over all ranks' copies, reduced INSIDE the NVSwitch -- a rank pulls P
// bytes instead of W * P, in one pass that also applies the update rule and writes the fp32 master weights.
//
// Set-up (driver VMM API, resolved through cudaGetDriverEntryPoint so the library has no link-time libcuda dependency):
//   rank 0:  cuMulticastCreate(numDevices = W, size)  ->  cuMemExportToShareableHandle (POSIX fd)  ->  fd travels to the peers over a
//            unix-domain socket (SCM_RIGHTS; parallel/p2p.py)
//   peers:   cuMemImportFromShareableHandle(fd)
//   all:     cuMulticastAddDevice;  [barrier];  cuMemCreate(local, POSIX fd type) + cuMulticastBindMem(mc, 0, local);
//            map local (unicast VA: where the backward writes gradients) and mc (multicast VA: what the all-reduce reads)
// Every step falls back to the P2P pull kernel when any of this is unavailable (dr_nvls_supported == 0).
#include <cuda.h>

#include "sp_sync.cuh"

using namespace drc;

namespace {

template <typename F> F drv(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
  return (F)p;
}
#define DRV(name) static auto p_##name = drv<decltype(&name)>(#name); if (!p_##name) return -900

struct NvlsState {
  CUmemGenericAllocationHandle mc = 0, mem = 0;
  CUdeviceptr local_va = 0, mc_va = 0;
  size_t size = 0;
  int dev = 0, world = 0;
};

size_t round_up(size_t n, size_t g) { return (n + g - 1) / g * g; }

CUmulticastObjectProp mc_prop(int world, size_t size) {
  CUmulticastObjectProp p = {};
  p.numDevices = (unsigned)world;
  p.size = size;
  p.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  p.flags = 0;
  return p;
}

// reduced = sum over ranks (in-switch) -> optimizer update, one pass.  mc: multicast VA of the symmetric gradient buffer.
__global__ void __launch_bounds__(256) k_nvls_allreduce_apply(const float* __restrict__ mc, float* __restrict__ w, float* __restrict__ s0,
                                                              float* __restrict__ s1, int64_t n4, const DrOptHyper* __restrict__ hp_dev,
                                                              float* __restrict__ reduced_out, DrSpSync sync) {
  pdl_sync();
  if (sync.state) sp_wait_all(sync, SP_CH_DENSE);       // every rank's gradients are complete and visible at system scope
  DrOptHyper hp = {};
  if (hp_dev) hp = *hp_dev;
  const float alpha = hp_dev ? dr_adam_alpha(hp) : 0.f;
  const bool decay_now = dr_dense_decay_now(hp);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 g;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(g.x), "=f"(g.y), "=f"(g.z), "=f"(g.w) : "l"(mc + 4 * i) : "memory");
    if (reduced_out) reinterpret_cast<float4*>(reduced_out)[i] = g;
    if (w) {
      float4 wv = reinterpret_cast<float4*>(w)[i];
      float4 a = s0 ? reinterpret_cast<float4*>(s0)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 b = s1 ? reinterpret_cast<float4*>(s1)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, g.x, wv.x, a.x, b.x);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, g.y, wv.y, a.y, b.y);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, g.z, wv.z, a.z, b.z);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, g.w, wv.w, a.w, b.w);
      reinterpret_cast<float4*>(w)[i] = wv;
      if (s0) reinterpret_cast<float4*>(s0)[i] = a;
      if (s1) reinterpret_cast<float4*>(s1)[i] = b;
    }
  }
}

// Two-phase variant for large gradients (the one-shot kernel makes every rank pull every element: W * P bytes leave each GPU, no better
// than the peer pull).  Phase A: rank r owns slice r -- ONE in-switch multimem.ld_reduce per 16 B of its slice, and ONE multimem.st that
// the switch fans out to every rank's buffer (the reduced value replaces the gradient in place; nobody else touches slice r).  Per GPU:
// P bytes out + P bytes in, independent of W.  Last block raises REDUCED; phase B (every rank) waits for all REDUCED flags and applies the
// optimizer from its LOCAL, now fully reduced, buffer.
constexpr int SP_CH_REDUCED = 5;
__global__ void __launch_bounds__(256) k_nvls_reduce_bcast(float* __restrict__ mc, int64_t n4, int rank, int W, DrSpSync sync) {
  pdl_sync();
  if (sync.state) sp_wait_all(sync, SP_CH_DENSE);
  const int64_t per = (n4 + W - 1) / W;
  const int64_t lo = per * rank, hi = min(n4, lo + per);
  for (int64_t i = lo + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    float4 g;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(g.x), "=f"(g.y), "=f"(g.z), "=f"(g.w) : "l"(mc + 4 * i) : "memory");
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + 4 * i), "f"(g.x), "f"(g.y), "f"(g.z), "f"(g.w) : "memory");
  }
  if (sync.state) sp_signal_last_block(sync, SP_CH_REDUCED);
}
__global__ void __launch_bounds__(256) k_nvls_apply_local(const float* __restrict__ g_local, float* __restrict__ w, float* __restrict__ s0,
                                                          float* __restrict__ s1, int64_t n4, const DrOptHyper* __restrict__ hp_dev, DrSpSync sync) {
  pdl_sync();
  if (sync.state) sp_wait_all(sync, SP_CH_REDUCED);      // every slice owner has broadcast its reduced slice into my buffer
  const DrOptHyper hp = *hp_dev;
  const float alpha = dr_adam_alpha(hp);
  const bool decay_now = dr_dense_decay_now(hp);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int4 raw = ld_v4_volatile(reinterpret_cast<const float4*>(g_local) + i);     // written by the switch: bypass L1
    const float4 g = make_float4(__int_as_float(raw.x), __int_as_float(raw.y), __int_as_float(raw.z), __int_as_float(raw.w));
    float4 wv = reinterpret_cast<float4*>(w)[i];
    float4 a = s0 ? reinterpret_cast<float4*>(s0)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 b = s1 ? reinterpret_cast<float4*>(s1)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    dr_apply_elem(hp.kind, hp, alpha, decay_now, g.x, wv.x, a.x, b.x);
    dr_apply_elem(hp.kind, hp, alpha, decay_now, g.y, wv.y, a.y, b.y);
    dr_apply_elem(hp.kind, hp, alpha, decay_now, g.z, wv.z, a.z, b.z);
    dr_apply_elem(hp.kind, hp, alpha, decay_now, g.w, wv.w, a.w, b.w);
    reinterpret_cast<float4*>(w)[i] = wv;
    if (s0) reinterpret_cast<float4*>(s0)[i] = a;
    if (s1) reinterpret_cast<float4*>(s1)[i] = b;
  }
}

}  // namespace

extern "C" {

// 1 when the device (and driver) support multicast objects.
int dr_nvls_supported(int dev) {
  DRV(cuDeviceGet); DRV(cuDeviceGetAttribute);
  CUdevice d;
  if (p_cuDeviceGet(&d, dev) != CUDA_SUCCESS) return 0;
  int ok = 0;
  if (p_cuDeviceGetAttribute(&ok, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, d) != CUDA_SUCCESS) return 0;
  return ok;
}

// granularity-rounded size every rank must use
int64_t dr_nvls_size(int64_t bytes, int world) {
  static auto p_gran = drv<decltype(&cuMulticastGetGranularity)>("cuMulticastGetGranularity");
  if (!p_gran) return -900;
  CUmulticastObjectProp p = mc_prop(world, (size_t)bytes);
  size_t g = 0;
  if (p_gran(&g, &p, CU_MULTICAST_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS || g == 0) return -901;
  return (int64_t)round_up((size_t)bytes, g);
}

// rank 0: create the multicast object and export it as a POSIX fd.  size = dr_nvls_size(...).
int dr_nvls_create(int64_t size, int world, int dev, void** out_state, int* out_fd) {
  DRV(cuMulticastCreate); DRV(cuMemExportToShareableHandle);
  DR_CUDA_CHECK(cudaSetDevice(dev));
  DR_CUDA_CHECK(cudaFree(0));
  auto* st = new NvlsState();
  st->size = (size_t)size; st->dev = dev; st->world = world;
  CUmulticastObjectProp p = mc_prop(world, (size_t)size);
  CUresult r = p_cuMulticastCreate(&st->mc, &p);
  if (r != CUDA_SUCCESS) { delete st; return -910 - (int)r; }
  int fd = -1;
  r = p_cuMemExportToShareableHandle(&fd, st->mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
  if (r != CUDA_SUCCESS) { delete st; return -920 - (int)r; }
  *out_state = st; *out_fd = fd;
  return 0;
}

// peers: import the multicast object from the fd received from rank 0.
int dr_nvls_import(int fd, int64_t size, int world, int dev, void** out_state) {
  DRV(cuMemImportFromShareableHandle);
  DR_CUDA_CHECK(cudaSetDevice(dev));
  DR_CUDA_CHECK(cudaFree(0));
  auto* st = new NvlsState();
  st->size = (size_t)size; st->dev = dev; st->world = world;
  CUresult r = p_cuMemImportFromShareableHandle(&st->mc, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
  if (r != CUDA_SUCCESS) { delete st; return -930 - (int)r; }
  *out_state = st;
  return 0;
}

// all ranks, phase 1 (before the host barrier): join the multicast team.
int dr_nvls_add_device(void* state) {
  DRV(cuDeviceGet); DRV(cuMulticastAddDevice);
  auto* st = static_cast<NvlsState*>(state);
  CUdevice d;
  if (p_cuDeviceGet(&d, st->dev) != CUDA_SUCCESS) return -940;
  CUresult r = p_cuMulticastAddDevice(st->mc, d);
  return r == CUDA_SUCCESS ? 0 : -950 - (int)r;
}

// all ranks, phase 2 (after every rank added its device): local physical memory, bind, map unicast + multicast VAs.
int dr_nvls_bind(void* state, void** local_ptr, void** mc_ptr) {
  DRV(cuMemCreate); DRV(cuMulticastBindMem); DRV(cuMemAddressReserve); DRV(cuMemMap); DRV(cuMemSetAccess);
  auto* st = static_cast<NvlsState*>(state);
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = st->dev;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUresult r = p_cuMemCreate(&st->mem, st->size, &prop, 0);
  if (r != CUDA_SUCCESS) return -960 - (int)r;
  r = p_cuMulticastBindMem(st->mc, 0, st->mem, 0, st->size, 0);
  if (r != CUDA_SUCCESS) return -970 - (int)r;
  CUmemAccessDesc acc = {};
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc.location.id = st->dev; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (p_cuMemAddressReserve(&st->local_va, st->size, 0, 0, 0) != CUDA_SUCCESS) return -980;
  if (p_cuMemMap(st->local_va, st->size, 0, st->mem, 0) != CUDA_SUCCESS) return -981;
  if (p_cuMemSetAccess(st->local_va, st->size, &acc, 1) != CUDA_SUCCESS) return -982;
  if (p_cuMemAddressReserve(&st->mc_va, st->size, 0, 0, 0) != CUDA_SUCCESS) return -983;
  if (p_cuMemMap(st->mc_va, st->size, 0, st->mc, 0) != CUDA_SUCCESS) return -984;
  if (p_cuMemSetAccess(st->mc_va, st->size, &acc, 1) != CUDA_SUCCESS) return -985;
  DR_CUDA_CHECK(cudaMemset((void*)st->local_va, 0, st->size));
  DR_CUDA_CHECK(cudaDeviceSynchronize());
  *local_ptr = (void*)st->local_va; *mc_ptr = (void*)st->mc_va;
  return 0;
}

// n multiple of 4.  w == null => pure all-reduce into reduced_out.  sync may be null (caller already synchronised the ranks).
int dr_nvls_allreduce_apply(const void* mc_ptr, float* w, float* s0, float* s1, int64_t n, const DrOptHyper* hp_dev, float* reduced_out,
                            const DrSpSync* sync, cudaStream_t s) {
  if (n % 4) return -2;
  int64_t b = (n / 4 + 255) / 256;
  if (b < 1) b = 1;
  if (b > num_sms() * 4) b = num_sms() * 4;
  DrSpSync sy{}; if (sync) sy = *sync;
  DR_PDL_LAUNCH((k_nvls_allreduce_apply), (int)b, 256, 0, s, (const float*)mc_ptr, w, s0, s1, n / 4, hp_dev, reduced_out, sy);
  DR_LAUNCH_CHECK();
  return 0;
}

// Two-phase NVLS all-reduce.  (a) reduce-scatter + multicast broadcast in place over the multicast mapping; with `w` given, (b) the optimizer
// from the local mapping follows (waits for every rank's REDUCED flag; `sync` required).  Without `w` the caller synchronises the ranks and
// reads its local buffer.
int dr_nvls_allreduce_2phase(void* mc_ptr, const float* local_ptr, int rank, int W, float* w, float* s0, float* s1, int64_t n,
                             const DrOptHyper* hp_dev, const DrSpSync* sync, cudaStream_t s) {
  if (n % 4) return -2;
  const int64_t n4 = n / 4, per = (n4 + W - 1) / W;
  int64_t b = (per + 255) / 256;
  if (b < 1) b = 1;
  if (b > num_sms() * 4) b = num_sms() * 4;
  DrSpSync sy{}; if (sync) sy = *sync;
  DR_PDL_LAUNCH((k_nvls_reduce_bcast), (int)b, 256, 0, s, (float*)mc_ptr, n4, rank, W, sy);
  DR_LAUNCH_CHECK();
  if (w) {
    if (!sync) return -3;
    int64_t b2 = (n4 + 255) / 256;
    if (b2 > num_sms() * 4) b2 = num_sms() * 4;
    DR_PDL_LAUNCH((k_nvls_apply_local), (int)b2, 256, 0, s, local_ptr, w, s0, s1, n4, hp_dev, sy);
    DR_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
