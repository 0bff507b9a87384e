// custom_cone.cuh -- convex cones whose projection the user writes in CUDA C++ (COSMO_B200_CUSTOM).
//
// The reference lets a user add a cone by subtyping AbstractConvexCone and defining project! (and optionally in_dual /
// in_pol_recc for the infeasibility certificates, convexset.jl:919-958).  Here the same three functions are CUDA device
// templates, with an optional fourth for the Jacobian of the projection: each type is compiled with NVRTC for sm_90a
// together with a small prelude and two or three generated wrapper kernels, loaded with cudaLibraryLoadData and launched
// on the engine stream like any other cone kernel.
//   cosmo_custom_project: copies a cone's w_s rows into s, synchronises the cone's lanes and calls NAME::project;
//   cosmo_custom_cert:    copies -v (primal certificate) or v (dual) into a scratch vector, calls the hook and writes
//                         flag[cone] = 0 when every lane certified, 1 otherwise; custom_flag_fold_kernel folds the flags
//                         of all types into one scalar in a fixed order;
//   cosmo_custom_jacobian: (types with COSMO_B200_CUSTOM_HAS_JACOBIAN) copies a cone's rows of a direction h into out,
//                         synchronises the lanes and calls NAME::jacobian(w_s, Pi(w_s), out): out = DPi(w_s) h, for
//                         the derivatives through the fixed point (solve_adjoint.cuh).
// The compiled cubins live in one process-wide cache keyed by the descriptor's contents and the dtype, so every engine
// (and every rank of a sharded model) of a process compiles a type once.  NVRTC is loaded with dlopen on first use, so
// that an engine without custom cones neither needs nor loads it.
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/cosmo_b200.h"
#include "host.cuh"

namespace cosmo {
namespace custom {

// ---- NVRTC through dlopen -----------------------------------------------------
typedef void* NvrtcProgram;
struct NvrtcApi {
  void* lib = nullptr;
  int (*CreateProgram)(NvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
  int (*CompileProgram)(NvrtcProgram, int, const char* const*) = nullptr;
  int (*GetProgramLogSize)(NvrtcProgram, size_t*) = nullptr;
  int (*GetProgramLog)(NvrtcProgram, char*) = nullptr;
  int (*GetCUBINSize)(NvrtcProgram, size_t*) = nullptr;
  int (*GetCUBIN)(NvrtcProgram, char*) = nullptr;
  int (*DestroyProgram)(NvrtcProgram*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  // called with the cache's mutex held
  void load() {
    if (lib) return;
    void* h = dlopen("libnvrtc.so.12", RTLD_NOW | RTLD_GLOBAL);
    if (!h) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, std::string("custom cones need NVRTC: cannot dlopen libnvrtc.so.12: ") + dlerror()};
    auto sym = [&](const char* s) {
      void* p = dlsym(h, s);
      if (!p) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, std::string("libnvrtc.so.12 lacks ") + s};
      return p;
    };
    CreateProgram = (decltype(CreateProgram))sym("nvrtcCreateProgram");
    CompileProgram = (decltype(CompileProgram))sym("nvrtcCompileProgram");
    GetProgramLogSize = (decltype(GetProgramLogSize))sym("nvrtcGetProgramLogSize");
    GetProgramLog = (decltype(GetProgramLog))sym("nvrtcGetProgramLog");
    GetCUBINSize = (decltype(GetCUBINSize))sym("nvrtcGetCUBINSize");
    GetCUBIN = (decltype(GetCUBIN))sym("nvrtcGetCUBIN");
    DestroyProgram = (decltype(DestroyProgram))sym("nvrtcDestroyProgram");
    GetErrorString = (decltype(GetErrorString))sym("nvrtcGetErrorString");
    lib = h;
  }
};

constexpr int kBlockLanes = 256;     // blockDim of a COSMO_B200_CUSTOM_BLOCK cone (and of the WARP launches)
constexpr int kThreadBlock = 128;    // blockDim of the THREAD launches

// Everything that makes two descriptors the same type for one dtype
struct Key {
  std::string name, source;
  int granularity = 0, n_params = 0, flags = 0, dtype = 0;
  bool operator<(const Key& o) const {
    return std::tie(name, source, granularity, n_params, flags, dtype) <
           std::tie(o.name, o.source, o.granularity, o.n_params, o.flags, o.dtype);
  }
};

// The checks of a descriptor that arrives through the C ABI (COSMO_B200_ERR_INVALID)
inline Key make_key(const cosmo_b200_custom_cone* d, int dtype) {
  if (!d) throw EngineError{COSMO_B200_ERR_INVALID, "custom cone: no type descriptor (set.u is NULL)"};
  if (!d->name || !d->source) throw EngineError{COSMO_B200_ERR_INVALID, "custom cone: name and source must be given"};
  const std::string name = d->name;
  bool ident = !name.empty() && !(name[0] >= '0' && name[0] <= '9');
  for (char c : name) ident = ident && ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_');
  if (!ident) throw EngineError{COSMO_B200_ERR_INVALID, "custom cone: name \"" + name + "\" is not a C identifier"};
  if (name == "cosmo_cone") throw EngineError{COSMO_B200_ERR_INVALID, "custom cone: the name cosmo_cone is the prelude's"};
  if (d->granularity < COSMO_B200_CUSTOM_THREAD || d->granularity > COSMO_B200_CUSTOM_BLOCK)
    throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + name + ": unknown granularity"};
  if (d->flags & ~(COSMO_B200_CUSTOM_HAS_IN_DUAL | COSMO_B200_CUSTOM_HAS_IN_POL_RECC | COSMO_B200_CUSTOM_HAS_JACOBIAN))
    throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + name + ": unknown flag"};
  if (d->reserved != 0) throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + name + ": reserved must be 0"};
  if (d->n_params < 0) throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + name + ": n_params < 0"};
  if (dtype != COSMO_B200_F64 && dtype != COSMO_B200_F32) throw EngineError{COSMO_B200_ERR_INVALID, "custom cone: dtype must be F64 or F32"};
  return Key{name, d->source, d->granularity, d->n_params, d->flags, dtype};
}

// Reductions over the lanes of one cone, for the user's code.  The block versions use shared memory and
// __syncthreads, so all lanes of the cone must call them; the sums run in a fixed order (deterministic).
static const char* kPrelude = R"PRELUDE(
namespace cosmo_cone {
template <typename T> __device__ __forceinline__ T max2_(T a, T b) { return b > a ? b : a; }
template <typename T> __device__ __forceinline__ T warp_sum(T v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <typename T> __device__ __forceinline__ T warp_max(T v) {
  for (int o = 16; o > 0; o >>= 1) v = max2_(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <typename T> __device__ T block_sum(T v) {
  __shared__ T sh[32];
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T r = sh[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r += sh[w];
  return r;
}
template <typename T> __device__ T block_max(T v) {
  __shared__ T sh[32];
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T r = sh[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = max2_(r, sh[w]);
  return r;
}
template <typename T> __device__ T sum(T v, int width) { return width == 1 ? v : width == 32 ? warp_sum(v) : block_sum(v); }
template <typename T> __device__ T max(T v, int width) { return width == 1 ? v : width == 32 ? warp_max(v) : block_max(v); }
__device__ inline bool all(bool b, int width) {
  return width == 1 ? b : width == 32 ? (__all_sync(0xffffffffu, b) != 0) : (__syncthreads_and(b) != 0);
}
__device__ inline void sync(int width) {
  if (width == 32) __syncwarp();
  else if (width > 32) __syncthreads();
}
}  // namespace cosmo_cone
)PRELUDE";

// The wrappers; COSMO_CONE_* are defined in front of the prelude
static const char* kWrappers = R"WRAP(
#define COSMO_CONE_LOCATE                                                                              \
  int cone, lane, width;                                                                               \
  if (COSMO_CONE_GRANULARITY == 0) { cone = blockIdx.x * blockDim.x + threadIdx.x; lane = 0; width = 1; } \
  else if (COSMO_CONE_GRANULARITY == 1) { cone = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; lane = threadIdx.x & 31; width = 32; } \
  else { cone = blockIdx.x; lane = threadIdx.x; width = blockDim.x; }                                  \
  if (cone >= ncones) return;                                                                          \
  const long long d = dim[cone];                                                                       \
  const COSMO_CONE_T* p = COSMO_CONE_NPARAMS ? params + (long long)cone * COSMO_CONE_NPARAMS : nullptr;

extern "C" __global__ void cosmo_custom_project(int ncones, const int* off, const int* dim, const COSMO_CONE_T* params,
                                                const COSMO_CONE_T* ws, COSMO_CONE_T* s) {
  COSMO_CONE_LOCATE
  COSMO_CONE_T* x = s + off[cone];
  const COSMO_CONE_T* w = ws + off[cone];
  for (long long i = lane; i < d; i += width) x[i] = w[i];
  cosmo_cone::sync(width);
  COSMO_CONE_NAME::project<COSMO_CONE_T>(x, d, p, lane, width);
}

// which = 0: in_dual(-v) (primal certificate), 1: in_pol_recc(v) (dual certificate)
extern "C" __global__ void cosmo_custom_cert(int ncones, const int* off, const int* dim, const COSMO_CONE_T* params,
                                             const COSMO_CONE_T* v, COSMO_CONE_T* tmp, COSMO_CONE_T tol, int which,
                                             int* flag) {
  COSMO_CONE_LOCATE
  COSMO_CONE_T* x = tmp + off[cone];
  const COSMO_CONE_T* src = v + off[cone];
  for (long long i = lane; i < d; i += width) x[i] = which == 0 ? -src[i] : src[i];
  cosmo_cone::sync(width);
  bool ok = false;
  if (which == 0) {
#if COSMO_CONE_FLAGS & 1
    ok = COSMO_CONE_NAME::in_dual<COSMO_CONE_T>(x, d, tol, p, lane, width);
#endif
  } else {
#if COSMO_CONE_FLAGS & 2
    ok = COSMO_CONE_NAME::in_pol_recc<COSMO_CONE_T>(x, d, tol, p, lane, width);
#endif
  }
  ok = cosmo_cone::all(ok, width);
  if (lane == 0) flag[cone] = ok ? 0 : 1;
}

#if COSMO_CONE_FLAGS & 8
// out = DPi(ws) h on the rows of every cone, ps = Pi(ws) at the same point
extern "C" __global__ void cosmo_custom_jacobian(int ncones, const int* off, const int* dim, const COSMO_CONE_T* params,
                                                 const COSMO_CONE_T* ws, const COSMO_CONE_T* ps, const COSMO_CONE_T* h,
                                                 COSMO_CONE_T* out) {
  COSMO_CONE_LOCATE
  COSMO_CONE_T* x = out + off[cone];
  const COSMO_CONE_T* src = h + off[cone];
  for (long long i = lane; i < d; i += width) x[i] = src[i];
  cosmo_cone::sync(width);
  COSMO_CONE_NAME::jacobian<COSMO_CONE_T>(ws + off[cone], ps + off[cone], x, d, p, lane, width);
}
#endif
)WRAP";

inline std::string generated_source(const Key& k) {
  std::string s;
  s += "#define COSMO_CONE_T " + std::string(k.dtype == COSMO_B200_F64 ? "double" : "float") + "\n";
  s += "#define COSMO_CONE_NAME " + k.name + "\n";
  s += "#define COSMO_CONE_GRANULARITY " + std::to_string(k.granularity) + "\n";
  s += "#define COSMO_CONE_NPARAMS " + std::to_string(k.n_params) + "\n";
  s += "#define COSMO_CONE_FLAGS " + std::to_string(k.flags) + "\n";
  s += kPrelude;
  s += "#line 1 \"" + k.name + "\"\n";
  s += k.source;
  s += "\n#line 1 \"cosmo_custom_wrappers\"\n";
  s += kWrappers;
  return s;
}

struct Entry {
  Key key;
  std::vector<char> cubin;
  cudaLibrary_t lib = nullptr;          // loaded on the first engine that uses the type (needs a device)
  cudaKernel_t project = nullptr, cert = nullptr;
  cudaKernel_t jac = nullptr;           // types with COSMO_B200_CUSTOM_HAS_JACOBIAN only
};

// One per process.  Entries are never removed or unloaded: a type compiled once stays usable by later engines.
class Cache {
 public:
  // The entry of `k`, compiled now when it is not cached yet (*compiled = true).
  Entry* get(const Key& k, bool* compiled) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = map_.find(k);
    if (it != map_.end()) { *compiled = false; return it->second.get(); }
    std::unique_ptr<Entry> e(new Entry());
    e->key = k;
    compile(*e);
    *compiled = true;
    Entry* p = e.get();
    map_[k] = std::move(e);
    return p;
  }
  // The kernels of `e`, loading its cubin on first use (the library is context independent: one load serves every device)
  void load(Entry* e) {
    std::lock_guard<std::mutex> g(mu_);
    if (e->lib) return;
    cudaLibrary_t lib = nullptr;
    CUDA_TRY(cudaLibraryLoadData(&lib, e->cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0));
    CUDA_TRY(cudaLibraryGetKernel(&e->project, lib, "cosmo_custom_project"));
    CUDA_TRY(cudaLibraryGetKernel(&e->cert, lib, "cosmo_custom_cert"));
    if (e->key.flags & COSMO_B200_CUSTOM_HAS_JACOBIAN) CUDA_TRY(cudaLibraryGetKernel(&e->jac, lib, "cosmo_custom_jacobian"));
    e->lib = lib;
  }

 private:
  std::mutex mu_;
  std::map<Key, std::unique_ptr<Entry>> map_;
  NvrtcApi nvrtc_;

  void compile(Entry& e) {
    nvrtc_.load();
    const std::string src = generated_source(e.key);
    NvrtcProgram prog = nullptr;
    int rc = nvrtc_.CreateProgram(&prog, src.c_str(), (e.key.name + ".cu").c_str(), 0, nullptr, nullptr);
    if (rc != 0) throw EngineError{COSMO_B200_ERR_INVALID, std::string("custom cone ") + e.key.name + ": nvrtcCreateProgram: " + nvrtc_.GetErrorString(rc)};
    // IEEE arithmetic as everywhere else in the engine: no fast-math flags
    const char* opts[] = {"-arch=sm_90a", "-std=c++17"};
    rc = nvrtc_.CompileProgram(prog, 2, opts);
    std::string log;
    size_t n = 0;
    if (nvrtc_.GetProgramLogSize(prog, &n) == 0 && n > 1) {
      log.resize(n);
      nvrtc_.GetProgramLog(prog, &log[0]);
      log.resize(n - 1);
    }
    if (rc == 0 && nvrtc_.GetCUBINSize(prog, &n) == 0) {
      e.cubin.resize(n);
      rc = nvrtc_.GetCUBIN(prog, e.cubin.data());
    }
    nvrtc_.DestroyProgram(&prog);
    if (rc != 0 || e.cubin.empty())
      throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + e.key.name + " does not compile (" + nvrtc_.GetErrorString(rc) + "):\n" + log};
  }
};

inline Cache& cache() {
  static Cache* c = new Cache();   // never destroyed: the CUDA runtime may be gone at process exit
  return *c;
}

inline void launch_dims(int granularity, int ncones, dim3& grid, dim3& block) {
  if (granularity == COSMO_B200_CUSTOM_THREAD) { block = dim3(kThreadBlock); grid = dim3((ncones + kThreadBlock - 1) / kThreadBlock); }
  else if (granularity == COSMO_B200_CUSTOM_WARP) { block = dim3(kBlockLanes); grid = dim3((ncones + kBlockLanes / 32 - 1) / (kBlockLanes / 32)); }
  else { block = dim3(kBlockLanes); grid = dim3(ncones); }
}

// The custom cones of one engine that share a type, as a slice of the engine's concatenated tables
struct TypeSlice {
  Entry* entry = nullptr;
  int first = 0, n = 0;        // cones [first, first + n) of the tables
  long long param_first = 0;   // first parameter of the type's first cone
};

}  // namespace custom

// OR of the per-cone certificate flags into one scalar (1: some cone is not certified); a single block, fixed order
template <typename T>
__global__ void __launch_bounds__(kBlock) custom_flag_fold_kernel(int n, const int* __restrict__ flag, T* __restrict__ out) {
  __shared__ int any;
  if (threadIdx.x == 0) any = 0;
  __syncthreads();
  int f = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) f |= flag[i];
  if (f) atomicOr(&any, 1);
  __syncthreads();
  if (threadIdx.x == 0) *out = any ? T(1) : T(0);
}

}  // namespace cosmo
