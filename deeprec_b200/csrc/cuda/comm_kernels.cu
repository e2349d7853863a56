// NVLink 5 / NVSwitch peer-memory layer: symmetric buffers (CUDA IPC), device-side rank barrier, and the
// fused compute+collective kernels of the model-parallel embedding / data-parallel dense step.
//
//   (the model-parallel embedding kernels live in sparse_pipeline.cu: k_sp_dedup / k_sp_lookup / k_sp_grad)
//   k_allreduce_apply   dense gradient all-reduce fused with the optimizer: every rank loads all peers' gradient
//                       shards over NVLink in a fixed order (bitwise identical sums on all ranks), applies the
//                       update rule and writes fp32 master weights in one pass.  Replaces Horovod ncclAllReduce +
//                       separate Apply* op (C1/K9).
//   k_rank_barrier      flag barrier over peer memory (st.release.sys / ld.acquire.sys), epoch kept on device so a
//                       captured CUDA graph replays it.
#include "sp_sync.cuh"
#include "table.cuh"

using namespace drc;

namespace {

constexpr int kMaxRanks = 16;

constexpr int kMaxChannels = 16;

// signals layout (per rank, symmetric): uint32 flags[kMaxChannels][kMaxRanks]; epochs[kMaxChannels] lives in LOCAL memory
__global__ void k_rank_barrier(DrPeers sig, uint32_t* __restrict__ epochs, int channel, int rank, int world) {
  pdl_sync();
  __shared__ uint32_t epoch;
  if (threadIdx.x == 0) { epoch = epochs[channel] + 1; epochs[channel] = epoch; }
  __syncthreads();
  const int r = threadIdx.x;
  if (r < world) {
    __threadfence_system();
    uint32_t* remote = reinterpret_cast<uint32_t*>(sig.ptr[r]) + channel * kMaxRanks + rank;
    st_release_sys(remote, epoch);
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(sig.ptr[rank]) + channel * kMaxRanks + r;
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) { __nanosleep(20); }
  }
}

// -----------------------------------------------------------------------------------------------------------------
// Dense all-reduce (one-shot over peer memory, fixed summation order) fused with the optimizer update.
// -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_allreduce_apply(DrPeers grad_peers, int W, float* __restrict__ w, float* __restrict__ s0,
                                                         float* __restrict__ s1, int64_t n4 /* n / 4 */, const DrOptHyper* __restrict__ hp_dev,
                                                         float* __restrict__ reduced_out, DrSpSync sync) {
  pdl_sync();
  if (sync.state) sp_wait_all(sync, SP_CH_DENSE);      // every rank's dense gradients are complete (flag raised by k_sp_signal)
  DrOptHyper hp = {};
  if (hp_dev) hp = *hp_dev;
  const float alpha = hp_dev ? dr_adam_alpha(hp) : 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < W; ++r) {
      int4 raw = ld_nc_v4(reinterpret_cast<const float4*>(grad_peers.ptr[r]) + i);
      g.x += __int_as_float(raw.x); g.y += __int_as_float(raw.y); g.z += __int_as_float(raw.z); g.w += __int_as_float(raw.w);
    }
    if (reduced_out) reinterpret_cast<float4*>(reduced_out)[i] = g;
    if (w) {
      float4 wv = reinterpret_cast<float4*>(w)[i];
      float4 a = s0 ? reinterpret_cast<float4*>(s0)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 b = s1 ? reinterpret_cast<float4*>(s1)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      dr_apply_elem(hp.kind, hp, alpha, false, g.x, wv.x, a.x, b.x);
      dr_apply_elem(hp.kind, hp, alpha, false, g.y, wv.y, a.y, b.y);
      dr_apply_elem(hp.kind, hp, alpha, false, g.z, wv.z, a.z, b.z);
      dr_apply_elem(hp.kind, hp, alpha, false, g.w, wv.w, a.w, b.w);
      reinterpret_cast<float4*>(w)[i] = wv;
      if (s0) reinterpret_cast<float4*>(s0)[i] = a;
      if (s1) reinterpret_cast<float4*>(s1)[i] = b;
    }
  }
}

inline int grid_for(int64_t n, int block, int max_blocks = num_sms() * 8) {
  int64_t b = (n + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

}  // namespace

extern "C" {

// ---- device / IPC plumbing (this library links its own static cudart: make its current device explicit) ----------
int dr_cuda_set_device(int dev) { DR_CUDA_CHECK(cudaSetDevice(dev)); return 0; }
int dr_cuda_set_sparse_blocks_per_sm(int n) { sparse_blocks_per_sm() = n < 1 ? 1 : n; return 0; }
int dr_cuda_get_device() { int d = -1; cudaGetDevice(&d); return d; }

int dr_comm_alloc(int64_t bytes, void** out) {
  DR_CUDA_CHECK(cudaMalloc(out, (size_t)bytes));
  DR_CUDA_CHECK(cudaMemset(*out, 0, (size_t)bytes));
  return 0;
}
int dr_comm_free(void* p) { DR_CUDA_CHECK(cudaFree(p)); return 0; }
int dr_comm_get_handle(void* p, void* handle64) {
  cudaIpcMemHandle_t h;
  DR_CUDA_CHECK(cudaIpcGetMemHandle(&h, p));
  memcpy(handle64, &h, sizeof(h));
  return 0;
}
int dr_comm_open_handle(const void* handle64, void** out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  DR_CUDA_CHECK(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
int dr_comm_close_handle(void* p) { DR_CUDA_CHECK(cudaIpcCloseMemHandle(p)); return 0; }
int dr_comm_can_access_peer(int dev, int peer) { int ok = 0; cudaDeviceCanAccessPeer(&ok, dev, peer); return ok; }

int dr_comm_barrier(const DrPeers* sig, uint32_t* epochs, int channel, int rank, int world, cudaStream_t s) {
  DR_PDL_LAUNCH((k_rank_barrier), 1, 32, 0, s, *sig, epochs, channel, rank, world);
  DR_LAUNCH_CHECK();
  return 0;
}

// n must be a multiple of 4.  w == null => pure all-reduce into reduced_out.
int dr_comm_allreduce_apply(const DrPeers* grad_peers, int W, float* w, float* s0, float* s1, int64_t n, const DrOptHyper* hp_dev,
                            float* reduced_out, cudaStream_t s) {
  if (n % 4) return -2;
  DR_PDL_LAUNCH((k_allreduce_apply), grid_for(n / 4, 256, num_sms() * 4), 256, 0, s, *grad_peers, W, w, s0, s1, n / 4, hp_dev, reduced_out, DrSpSync{});
  DR_LAUNCH_CHECK();
  return 0;
}
// same, but the kernel itself waits for every rank's DENSE flag (no barrier kernel in front of it)
int dr_comm_allreduce_apply_sync(const DrPeers* grad_peers, int W, float* w, float* s0, float* s1, int64_t n, const DrOptHyper* hp_dev,
                                 float* reduced_out, const DrSpSync* sync, cudaStream_t s) {
  if (n % 4) return -2;
  DR_PDL_LAUNCH((k_allreduce_apply), grid_for(n / 4, 256, num_sms() * 4), 256, 0, s, *grad_peers, W, w, s0, s1, n / 4, hp_dev, reduced_out, *sync);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
