// SM partition of one device into two green contexts: a "sparse" one of R SMs and a "dense" one with the SMs left over, one stream in each.
//
// The DLRM step runs its embedding branch beside the bottom MLP.  Two streams of one context do not share the machine that way: a
// persistent wgmma GEMM needs a whole SM (up to 384 threads x 168 registers and ~200 KB of shared memory), so an SM holding a few sparse
// blocks takes no GEMM CTA, and the two streams end up time-slicing whole SMs.  Green contexts give each stream its own SMs, and a
// kernel node captured from a green-context stream keeps that context in the graph.
//
// Driver API resolved through cudaGetDriverEntryPoint, like nvls.cu: the library keeps no link-time libcuda dependency.
// Hopper splits SMs in groups of 8, so R is rounded; the caller gets the counts the driver actually provisioned.
#include <cuda.h>
#include <cuda_runtime.h>

#include <mutex>
#include <vector>

namespace {

template <typename F> F drv(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
  return (F)p;
}
#define DRV(name) static auto p_##name = drv<decltype(&name)>(#name); if (!p_##name) return -900
#define CK(call) do { CUresult r_ = (call); if (r_ != CUDA_SUCCESS) return -(int)r_; } while (0)

struct Side {
  CUgreenCtx g = nullptr;
  CUcontext ctx = nullptr;        // the green context as a CUcontext: what a captured kernel node records
  CUstream stream = nullptr;
  int sms = 0;
};

struct Partition {
  int device = -1, requested = -1;
  CUcontext primary = nullptr;
  Side sparse, dense;
};

std::mutex g_mu;
std::vector<Partition*> g_parts;  // created once per (device, requested SMs) and kept for the life of the process

int make_side(CUdevice dev, CUdevResource* res, Side* s) {
  DRV(cuDevResourceGenerateDesc); DRV(cuGreenCtxCreate); DRV(cuCtxFromGreenCtx); DRV(cuGreenCtxStreamCreate);
  CUdevResourceDesc desc = nullptr;
  CK(p_cuDevResourceGenerateDesc(&desc, res, 1));
  CK(p_cuGreenCtxCreate(&s->g, desc, dev, CU_GREEN_CTX_DEFAULT_STREAM));
  CK(p_cuCtxFromGreenCtx(&s->ctx, s->g));
  CK(p_cuGreenCtxStreamCreate(&s->stream, s->g, CU_STREAM_NON_BLOCKING, 0));
  s->sms = (int)res->sm.smCount;
  return 0;
}

int create(int device, int sparse_sms, Partition** out) {
  DRV(cuDeviceGet); DRV(cuDeviceGetDevResource); DRV(cuDevSmResourceSplitByCount); DRV(cuCtxGetCurrent);
  std::lock_guard<std::mutex> lk(g_mu);
  for (Partition* p : g_parts)
    if (p->device == device && p->requested == sparse_sms) { *out = p; return 0; }
  int cur = 0;
  if (cudaGetDevice(&cur) != cudaSuccess || cur != device || cudaFree(nullptr) != cudaSuccess) return -901;   // primary context current
  CUcontext primary = nullptr;
  CK(p_cuCtxGetCurrent(&primary));
  CUdevice dev;
  CK(p_cuDeviceGet(&dev, device));
  CUdevResource all{}, sparse{}, rest{};
  CK(p_cuDeviceGetDevResource(dev, &all, CU_DEV_RESOURCE_TYPE_SM));
  unsigned int groups = 1;
  CK(p_cuDevSmResourceSplitByCount(&sparse, &groups, &all, &rest, 0, (unsigned)sparse_sms));
  if (groups != 1 || rest.sm.smCount == 0) return -902;
  Partition* p = new Partition;
  p->device = device;
  p->requested = sparse_sms;
  p->primary = primary;
  int rc = make_side(dev, &sparse, &p->sparse);
  if (rc == 0) rc = make_side(dev, &rest, &p->dense);
  if (rc != 0) { delete p; return rc; }                          // a half-made partition is leaked to the driver, never handed out
  g_parts.push_back(p);
  *out = p;
  return 0;
}

}  // namespace

extern "C" {

// Partition `device` into a green context of (about) `sparse_sms` SMs and one of the remaining SMs.  Returns 0 and fills
// info[0..1] = SMs the sparse / dense context got, handles[0..1] = their streams, handles[2..4] = the sparse, dense and primary
// contexts as CUcontext.  `device` must be the current device.  Returns a negative CUresult (or -90x) when the driver refuses.
int dr_cuda_sm_partition(int device, int sparse_sms, int* info, void** handles) {
  if (sparse_sms <= 0) return -2;
  Partition* p = nullptr;
  int rc = create(device, sparse_sms, &p);
  if (rc != 0) return rc;
  info[0] = p->sparse.sms;
  info[1] = p->dense.sms;
  handles[0] = p->sparse.stream; handles[1] = p->dense.stream;
  handles[2] = p->sparse.ctx;    handles[3] = p->dense.ctx;    handles[4] = p->primary;
  return 0;
}

// The context of every kernel node of `graph` (a cudaGraph_t), in node order: up to `cap` handles into ctx_out.  Returns the number of
// kernel nodes, or a negative error.
int dr_cuda_graph_kernel_contexts(void* graph, void** ctx_out, int cap) {
  DRV(cuGraphGetNodes); DRV(cuGraphNodeGetType); DRV(cuGraphKernelNodeGetParams);
  size_t n = 0;
  CK(p_cuGraphGetNodes((CUgraph)graph, nullptr, &n));
  std::vector<CUgraphNode> nodes(n);
  CK(p_cuGraphGetNodes((CUgraph)graph, nodes.data(), &n));
  int k = 0;
  for (size_t i = 0; i < n; ++i) {
    CUgraphNodeType t;
    CK(p_cuGraphNodeGetType(nodes[i], &t));
    if (t != CU_GRAPH_NODE_TYPE_KERNEL) continue;
    CUDA_KERNEL_NODE_PARAMS kp{};
    CK(p_cuGraphKernelNodeGetParams(nodes[i], &kp));
    if (k < cap) ctx_out[k] = kp.ctx;
    ++k;
  }
  return k;
}

}  // extern "C"
