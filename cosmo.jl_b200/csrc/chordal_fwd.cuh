// chordal_fwd.cuh -- the way forward through a chordal decomposition for values: P, A, q and b of the original problem
// mapped onto the decomposed (clique) problem the engine holds (cosmo_b200_update_matrices_original).
//
// The decomposition is a function of the sparsity pattern, so the map is computed once on the host
// (chordal.forward_arrays) and handed over with cosmo_b200_set_forward_map:
//   A' (sorted CSC order, the order of At_.val): entry k is Ax[a_src[k]], +1.0 for a_src[k] = -1, -1.0 for -2 (the
//      overlap columns); every entry of A is used exactly once, no sums;
//   b': b'[i] = b[b_src[i]] for a plain row, 0.0 for b_src[i] = -1, and b[-2 - b_src[i]] for a row of a clique block,
//      where a zero of either sign arrives as +0.0 (the host decomposition writes only the nonzero values there);
//   q' = [q; 0];  P' has P's values in P's order.
// A row of a decomposed cone that lies in no clique has no place in b': a b that is nonzero there changes the
// aggregate pattern.  count_uncovered finds such rows on the device before anything is written.
// The maps are kept as int32 where every index fits, as the value maps of mat_update.cuh are.
// Included from engine.cu (after common.cuh).
#pragma once
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/cosmo_b200.h"
#include "host.cuh"

namespace cosmo {
namespace fwd {

// out[k] = v[src[k]], +1 for src[k] = -1, -1 for src[k] = -2
template <typename T, typename I>
__global__ void __launch_bounds__(kBlock) fwd_values_kernel(long long n, const I* __restrict__ src, const T* __restrict__ v,
                                                            T* __restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const I s = src[k];
    out[k] = s >= 0 ? v[s] : (s == -1 ? T(1) : T(-1));
  }
}

// out[i] = b[src[i]]; 0 for src[i] = -1; b[-2 - src[i]] with -0.0 -> +0.0 below that.  With E: out[i] = O(E[i] * that),
// the product taken in fp64 (update!(b=) of an original-coordinate fp64 b on a scaled engine)
template <typename T, typename I, typename O>
__global__ void __launch_bounds__(kBlock) fwd_b_kernel(long long m, const I* __restrict__ src, const T* __restrict__ b,
                                                       const O* __restrict__ E, O* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
    const I s = src[i];
    T v;
    if (s >= -1) {
      v = s >= 0 ? b[s] : T(0);
    } else {
      v = b[-2 - s];
      if (v == T(0)) v = T(0);
    }
    out[i] = E ? O((double)E[i] * (double)v) : O(v);
  }
}

// Rows of b that are nonzero (NaN counts) where `uncovered` is set, in two stages without atomics: one count per block,
// then fwd_count_sum_kernel adds them in block order.
template <typename T>
__global__ void __launch_bounds__(kBlock) fwd_b_check_kernel(long long m, const T* __restrict__ b,
                                                             const unsigned char* __restrict__ uncovered,
                                                             unsigned long long* __restrict__ partial) {
  __shared__ unsigned long long warp_cnt[kBlock / 32];
  unsigned long long c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x)
    c += (uncovered[i] && !(b[i] == T(0))) ? 1ull : 0ull;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < kBlock / 32; ++w) t += warp_cnt[w];
    partial[blockIdx.x] = t;
  }
}
__global__ void fwd_count_sum_kernel(int nblocks, const unsigned long long* __restrict__ partial,
                                     unsigned long long* __restrict__ total) {
  unsigned long long t = 0;
  for (int k = 0; k < nblocks; ++k) t += partial[k];
  *total = t;
}

static inline int grid_for(long long work) {
  return (int)std::min<long long>(std::max<long long>((work + kBlock - 1) / kBlock, 1), kMaxGrid);
}

// The forward map of one engine, validated, on the device.
class Forward {
 public:
  bool has_map() const { return set_; }
  int64_t n_orig() const { return n_orig_; }
  int64_t m_orig() const { return m_orig_; }
  int64_t nnzA_orig() const { return nnzA_orig_; }

  void clear() {
    set_ = false;
    a32_.release(); b32_.release(); a64_.release(); b64_.release(); unc_.release();
  }

  // n, m, nnzA: the engine's (decomposed) problem
  void set(const cosmo_b200_forward_map& f, int64_t n, int64_t m, int64_t nnzA, cudaStream_t st) {
    clear();
    auto bad = [](const std::string& msg) { throw EngineError{COSMO_B200_ERR_INVALID, "forward map: " + msg}; };
    if (f.n != n || f.m != m || f.nnzA != nnzA)
      bad("n, m, nnzA (" + std::to_string(f.n) + ", " + std::to_string(f.m) + ", " + std::to_string(f.nnzA) +
          ") are not the engine's (" + std::to_string(n) + ", " + std::to_string(m) + ", " + std::to_string(nnzA) + ")");
    if (f.n_orig < 0 || f.n_orig > n || f.m_orig < 0 || f.nnzA_orig < 0 || (nnzA && !f.a_src) || (m && !f.b_src) ||
        (f.m_orig && !f.b_uncovered))
      bad("bad dimensions or a missing array");
    std::vector<unsigned char> used((size_t)std::max(f.nnzA_orig, f.m_orig), 0);
    int64_t n_used = 0;
    for (int64_t k = 0; k < nnzA; ++k) {
      const int64_t s = f.a_src[k];
      if (s < -2 || s >= f.nnzA_orig) bad("a_src[" + std::to_string(k) + "] is out of range");
      if (s < 0) continue;
      if (used[s]) bad("entry " + std::to_string(s) + " of A is used twice");
      used[s] = 1;
      ++n_used;
    }
    if (n_used != f.nnzA_orig) bad("an entry of A is not used");
    std::fill(used.begin(), used.end(), 0);
    for (int64_t i = 0; i < m; ++i) {
      const int64_t s = f.b_src[i] < -1 ? -2 - f.b_src[i] : f.b_src[i];   // the source row; -1: none
      if (s >= f.m_orig) bad("b_src[" + std::to_string(i) + "] is out of range");
      if (s < 0) continue;
      if (used[s]) bad("row " + std::to_string(s) + " of b is used twice");
      used[s] = 1;
    }
    for (int64_t i = 0; i < f.m_orig; ++i)
      if ((used[i] != 0) == (f.b_uncovered[i] != 0))
        bad("row " + std::to_string(i) + " of b is " + (used[i] ? "used and marked uncovered" : "neither used nor marked uncovered"));

    n_orig_ = f.n_orig; m_orig_ = f.m_orig; nnzA_orig_ = f.nnzA_orig; n_ = n; m_ = m; nnzA_ = nnzA;
    wide_ = std::max(f.nnzA_orig, f.m_orig + 2) > (int64_t)INT32_MAX;
    if (wide_) {
      a64_.alloc(std::max<int64_t>(nnzA, 1), false); a64_.upload(f.a_src, nnzA, st);
      b64_.alloc(std::max<int64_t>(m, 1), false); b64_.upload(f.b_src, m, st);
    } else {
      std::vector<int> a(f.a_src, f.a_src + nnzA), b(f.b_src, f.b_src + m);
      a32_.alloc(std::max<int64_t>(nnzA, 1), false); a32_.upload(a.data(), a.size(), st);
      b32_.alloc(std::max<int64_t>(m, 1), false); b32_.upload(b.data(), b.size(), st);
      CUDA_TRY(cudaStreamSynchronize(st));   // the narrowed copies are locals
    }
    unc_.alloc(std::max<int64_t>(f.m_orig, 1), false);
    unc_.upload(f.b_uncovered, f.m_orig, st);
    partial_.alloc(kMaxGrid + 1, false);
    CUDA_TRY(cudaStreamSynchronize(st));
    set_ = true;
  }

  // rows of `b` (device, m_orig) that are nonzero outside every clique
  template <typename T>
  long long count_uncovered(const T* b, cudaStream_t st) {
    if (m_orig_ == 0) return 0;
    const int grid = grid_for(m_orig_);
    fwd_b_check_kernel<T><<<grid, kBlock, 0, st>>>(m_orig_, b, unc_.p, partial_.p);
    fwd_count_sum_kernel<<<1, 1, 0, st>>>(grid, partial_.p, partial_.p + kMaxGrid);
    CUDA_TRY(cudaGetLastError());
    unsigned long long total = 0;
    CUDA_TRY(cudaMemcpyAsync(&total, partial_.p + kMaxGrid, sizeof(total), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return (long long)total;
  }

  // the values of A' (nnzA, sorted CSC order) from the staged values of A (device, nnzA_orig)
  template <typename T>
  void gather_values(const T* ax, T* out, cudaStream_t st) {
    if (wide_) fwd_values_kernel<T, int64_t><<<grid_for(nnzA_), kBlock, 0, st>>>(nnzA_, a64_.p, ax, out);
    else fwd_values_kernel<T, int><<<grid_for(nnzA_), kBlock, 0, st>>>(nnzA_, a32_.p, ax, out);
    CUDA_TRY(cudaGetLastError());
  }

  // b' (m) from the staged b (device, m_orig), times E when E is not null
  template <typename T, typename O = T>
  void gather_b(const T* b, O* out, cudaStream_t st, const O* E = nullptr) {
    if (wide_) fwd_b_kernel<T, int64_t, O><<<grid_for(m_), kBlock, 0, st>>>(m_, b64_.p, b, E, out);
    else fwd_b_kernel<T, int, O><<<grid_for(m_), kBlock, 0, st>>>(m_, b32_.p, b, E, out);
    CUDA_TRY(cudaGetLastError());
  }

 private:
  bool set_ = false, wide_ = false;
  int64_t n_orig_ = 0, m_orig_ = 0, nnzA_orig_ = 0, n_ = 0, m_ = 0, nnzA_ = 0;
  DevBuf<int> a32_, b32_;
  DevBuf<int64_t> a64_, b64_;
  DevBuf<unsigned char> unc_;
  DevBuf<unsigned long long> partial_;   // one count per block, then the total
};

}  // namespace fwd
}  // namespace cosmo
