// host.cuh -- how the engine's host code owns CUDA resources and reports failures.
//
// Every failure is an EngineError carrying the COSMO_B200_ERR_* code the C ABI returns.  The owning types are
// non-copyable, start empty, are allocated or created explicitly (after the engine has selected its device) and free
// their resource in the destructor.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include <string>
#include <utility>
#include <vector>

#include "../../include/cosmo_b200.h"

namespace cosmo {

struct EngineError {
  int code;
  std::string msg;
};

#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      char _b[512];                                                                                 \
      snprintf(_b, sizeof(_b), "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__,        \
               __LINE__, cudaGetErrorString(_e));                                                   \
      throw EngineError{COSMO_B200_ERR_CUDA, _b};                                                   \
    }                                                                                               \
  } while (0)

// A failed allocation throws ERR_ALLOC.  Its error is taken off the runtime's last-error record, so that the next
// launch check does not report it a second time (a caller may carry on with less memory).
template <typename U>
struct DevBuf {
  U* p = nullptr;
  size_t n = 0;
  DevBuf() {} DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  void alloc(size_t count, bool zero = true) {
    if (p) { cudaFree(p); p = nullptr; }
    n = 0;
    size_t bytes = (count + 8) * sizeof(U);   // +8: bulk (TMA) copies round the tail up to 16 bytes
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
      p = nullptr;
      throw EngineError{COSMO_B200_ERR_ALLOC, std::string("cudaMalloc failed: ") + cudaGetErrorString(cudaGetLastError())};
    }
    n = count;
    if (zero) {
      // cudaMemset runs on the legacy default stream, which does NOT order against the engine's
      // non-blocking stream: wait for it here or a later kernel may race with the pending fill.
      CUDA_TRY(cudaMemset(p, 0, bytes));
      CUDA_TRY(cudaDeviceSynchronize());
    }
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  void upload(const U* host, size_t count, cudaStream_t st) {
    if (count) CUDA_TRY(cudaMemcpyAsync(p, host, count * sizeof(U), cudaMemcpyDefault, st));
  }
  void upload(const std::vector<U>& h, cudaStream_t st) {
    if (n < h.size()) alloc(h.size(), false);
    upload(h.data(), h.size(), st);
  }
};

// page-locked host memory: the mirrors that device scalars are read back into
template <typename U>
struct PinnedBuf {
  U* p = nullptr;
  PinnedBuf() {} PinnedBuf(const PinnedBuf&) = delete; PinnedBuf& operator=(const PinnedBuf&) = delete;
  ~PinnedBuf() { if (p) cudaFreeHost(p); }
  void alloc(size_t count) {
    if (p) { cudaFreeHost(p); p = nullptr; }
    if (cudaMallocHost(&p, count * sizeof(U)) != cudaSuccess) {
      p = nullptr;
      throw EngineError{COSMO_B200_ERR_ALLOC, std::string("cudaMallocHost failed: ") + cudaGetErrorString(cudaGetLastError())};
    }
  }
  U& operator[](size_t i) const { return p[i]; }
};

struct Event {
  cudaEvent_t e = nullptr;
  Event() {} Event(const Event&) = delete; Event& operator=(const Event&) = delete;
  ~Event() { if (e) cudaEventDestroy(e); }
  void create() { if (!e) CUDA_TRY(cudaEventCreate(&e)); }
  operator cudaEvent_t() const { return e; }
};

struct GraphExec {
  cudaGraphExec_t g = nullptr;
  GraphExec() {} GraphExec(const GraphExec&) = delete; GraphExec& operator=(const GraphExec&) = delete;
  ~GraphExec() { reset(); }
  void reset() { if (g) cudaGraphExecDestroy(g); g = nullptr; }
  operator cudaGraphExec_t() const { return g; }
};

// Launch `kernel` on `st` as a programmatic dependent of the kernel before it: it may be scheduled as soon as that kernel
// calls pdl_launch_dependents() (common.cuh), and must itself call pdl_wait() before it touches anything an earlier kernel
// of the stream reads or writes.  Stream capture records the programmatic edge in the graph.
template <typename... KArgs, typename... Args>
void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
}

// Stream-capture what `launches()` enqueues on `st` into `out`.
template <typename F>
void capture_graph(GraphExec& out, cudaStream_t st, F&& launches) {
  out.reset();
  cudaGraph_t graph = nullptr;
  CUDA_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  launches();
  CUDA_TRY(cudaStreamEndCapture(st, &graph));
  CUDA_TRY(cudaGraphInstantiate(&out.g, graph, 0));
  CUDA_TRY(cudaGraphDestroy(graph));
}

}  // namespace cosmo
