// common.cuh -- shared device helpers for the COSMO H100 engine (sm_90a).
//
// * streaming 128-bit loads for the CSR value / index streams (read once per
//   SpMV: keep them out of L1 so the gathered vector stays resident),
// * a deterministic multi-output block reduction with a "last block" second
//   stage: every kernel that produces scalars (dots, norms, inf-norms) writes
//   per-block partials, the last block to finish folds them in a fixed order
//   and runs a tiny scalar epilogue (the `finalize` functor).  No floating-point
//   atomics anywhere => bitwise reproducible runs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <limits>

namespace cosmo {

constexpr int kBlock = 256;           // threads per block for every reducing kernel
constexpr int kWarpsPerBlock = kBlock / 32;
constexpr int kMaxGrid = 132 * 8;     // 132 SMs x 8 resident 256-thread blocks
constexpr int kMaxRed = 8;            // max reduction slots per kernel

// grid of a kBlock-thread grid-stride loop over n elements
inline int vgrid(long long n) { return (int)std::min<long long>(std::max<long long>((n + kBlock - 1) / kBlock, 1), kMaxGrid); }

template <typename T>
struct CsrView {
  const int* rowptr;  // nrows+1 (nullptr => matrix absent)
  const int* col;
  const T* val;
};

// per-stream scratch for the two-stage reductions
template <typename T>
struct RedBuf {
  T* partials;        // kMaxGrid * kMaxRed
  T* out;             // where the folded scalars go (NS sums then NM maxes)
  unsigned* ticket;   // zero between kernels
};

// ---- streaming loads --------------------------------------------------------
__device__ __forceinline__ void load4_stream(const double* p, double (&v)[4]) {
  double2 a = __ldcs(reinterpret_cast<const double2*>(p));
  double2 b = __ldcs(reinterpret_cast<const double2*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void load4_stream(const float* p, float (&v)[4]) {
  float4 a = __ldcs(reinterpret_cast<const float4*>(p));
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
__device__ __forceinline__ int4 load4_stream(const int* p) {
  return __ldcs(reinterpret_cast<const int4*>(p));
}
// One lane's 8 values of a windowed row-segment step.  Values are stored "instruction-coalesced":
// the k-th 16-byte load of lane l sits at base + k * (EPL * L) + l * EPL  (EPL = elements per 16 B,
// L = active lanes of the step), so every load instruction of the warp covers one contiguous run of
// L * 16 bytes -- each 32-byte sector is requested exactly once.
__device__ __forceinline__ void load8_coalesced(const double* base, int L, int lane, double (&v)[8]) {
  const double2* q = reinterpret_cast<const double2*>(base) + lane;
  const double2 a = __ldcs(q), b = __ldcs(q + L), c = __ldcs(q + 2 * L), d = __ldcs(q + 3 * L);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void load8_coalesced(const float* base, int L, int lane, float (&v)[8]) {
  const float4* q = reinterpret_cast<const float4*>(base) + lane;
  const float4 a = __ldcs(q), b = __ldcs(q + L);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// ---- mbarrier + 1-D bulk (TMA) copy global -> shared ------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_load_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (unsigned)__cvta_generic_to_shared(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  const unsigned addr = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(addr),
      "r"(parity)
      : "memory");
}

// ---- programmatic dependent launch (launch_pdl in host.cuh) -----------------
// A kernel launched with launch_pdl may start while the kernel before it in the stream is still running.  Until
// pdl_wait() returns it may touch only data that stay constant during the solve (matrix slabs, row partitions, shape
// arguments): pdl_wait() blocks until every earlier kernel of the stream has completed and its writes are visible.
// Without a programmatic predecessor (first launch, after a collective, a copy or an event) it returns at once.
// pdl_launch_dependents() lets the next launch_pdl kernel start being scheduled; its CTAs take SMs as ours leave.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- peer-memory exchange (NVLink / NVSwitch) -------------------------------
// One exchange buffer per rank, mapped into every peer through CUDA IPC:
//   data : 2 slots x stride elements (the rank's partial n-vector + its partial dot at [n])
//   flags: 2 slots x kMaxRanks sequence numbers, written REMOTELY by the producers
// A producer writes its partial into its own slot (seq & 1) and publishes seq+1 into every peer's
// flag array; a consumer waits until all ranks have published seq+1, then sums the peers' slots in
// rank order while it does its own work (one-shot allreduce fused into the consumer kernel; the
// result is bitwise identical on every rank).  Two slots suffice: a rank can only overwrite slot s
// after all peers have published the NEXT sequence number, i.e. finished reading slot s.
constexpr int kMaxRanks = 8;
template <typename T>
struct P2pView {
  T* peer_data[kMaxRanks];         // peer_data[r] = base of rank r's exchange buffer (own buffer at r = rank); PUSH model:
                                   // rank q stores its partial into segment (slot * nranks + q) of EVERY rank's buffer,
                                   // consumers read their own buffer only
  unsigned* peer_flags[kMaxRanks]; // peer_flags[r] = base of rank r's flag array (remote writes)
  const unsigned* local_flags;     // this rank's flag array
  unsigned* seq;                   // device-resident sequence counter (identical on every rank)
  size_t stride;                   // elements per slot
  int nranks, rank;
};
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
template <typename T>
__device__ __forceinline__ T ld_peer(const T* p) {   // coherent load of peer / own exchange data
  return *reinterpret_cast<const volatile T*>(p);
}
// consumer side: block-wide wait until every rank has published sequence number `want` for `slot`
template <typename T>
__device__ __forceinline__ void p2p_wait_all(const P2pView<T>& v, unsigned slot, unsigned want) {
  if ((int)threadIdx.x < v.nranks) {
    const unsigned* f = v.local_flags + slot * kMaxRanks + threadIdx.x;
    while (ld_acquire_sys(f) != want) { __nanosleep(40); }
  }
  __syncthreads();
}
// producer side (one thread, after the kernel's data is globally visible): publish to all peers
template <typename T>
__device__ __forceinline__ void p2p_publish(const P2pView<T>& v, unsigned slot, unsigned val) {
  __threadfence_system();
  for (int r = 0; r < v.nranks; ++r) st_release_sys(v.peer_flags[r] + slot * kMaxRanks + v.rank, val);
}

// NaN-propagating max of non-negative magnitudes (Julia's norm(x, Inf) returns NaN
// when an entry is NaN; fmax would silently drop it).
template <typename T>
__device__ __forceinline__ T nanmax(T a, T b) {
  return (a > b || a != a) ? a : b;
}

template <typename T>
__device__ __forceinline__ T tabs(T a) { return a < 0 ? -a : a; }

// exponent e with |x| < 2^e for the largest |x| of a block (0 for 0, inf or NaN), clamped so that 2^-e and 2^e are both
// normal numbers of T: scaling by 2^-e is exact and brings the maximum into [0.5, 1)
template <typename T>
__device__ __forceinline__ int pow2_exponent(T mx) {
  constexpr double kMax = sizeof(T) == 8 ? 1.7976931348623157e308 : 3.4028234663852886e38;
  constexpr int lim = std::numeric_limits<T>::max_exponent - 2;
  int e = 0;
  if (mx > T(0) && (double)mx <= kMax) frexp((double)mx, &e);
  return e < -lim ? -lim : (e > lim ? lim : e);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <typename T>
__device__ __forceinline__ T warp_nanmax(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nanmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Fold per-thread accumulators (NS sums, NM maxes) over the block, publish the
// block partial, and let the last block fold all partials and call fin(out).
// Must be called by all kBlock threads of every block of the grid.
// `slot` / `nslots`: position of this block's partial and the number of participating blocks
// (default: every block of the grid, indexed by blockIdx.x).
// MAXR: slots per block the partials buffer of `rb` holds (kMaxRed for the engine's shared buffer).
template <typename T, int NS, int NM, typename Fin, int NWARPS = kWarpsPerBlock, int MAXR = kMaxRed>
__device__ __forceinline__ void reduce_and_finalize(const T* accS, const T* accM, const RedBuf<T>& rb,
                                                    const Fin& fin, int slot = -1, int nslots = -1) {
  if (slot < 0) { slot = blockIdx.x; nslots = gridDim.x; }
  constexpr int NR = NS + NM;
  static_assert(NR >= 1 && NR <= MAXR, "reduction slots");
  __shared__ T sm[NWARPS][NR];
  __shared__ int is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NS; ++k) {
    T v = warp_sum(accS[k]);
    if (lane == 0) sm[warp][k] = v;
  }
#pragma unroll
  for (int k = 0; k < NM; ++k) {
    T v = warp_nanmax(accM[k]);
    if (lane == 0) sm[warp][NS + k] = v;
  }
  __syncthreads();
  if (threadIdx.x < NR) {
    const int k = threadIdx.x;
    T v = sm[0][k];
    for (int w = 1; w < NWARPS; ++w) v = (k < NS) ? v + sm[w][k] : nanmax(v, sm[w][k]);
    rb.partials[(size_t)slot * NR + k] = v;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = atomicAdd(rb.ticket, 1u);
    is_last = (t == (unsigned)nslots - 1u);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    for (int k = warp; k < NR; k += NWARPS) {
      T v = 0;
      for (int b = lane; b < nslots; b += 32) {
        T p = __ldcg(rb.partials + (size_t)b * NR + k);
        v = (k < NS) ? v + p : nanmax(v, p);
      }
      v = (k < NS) ? warp_sum(v) : warp_nanmax(v);
      if (lane == 0) rb.out[k] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      fin(rb.out);
      *rb.ticket = 0u;
    }
  }
}

struct NoFin {
  template <typename T>
  __device__ void operator()(T*) const {}
};

}  // namespace cosmo
