// ldl.cuh -- direct LDL' solve of the quasi-definite KKT system K [y1; y2] = [x1; x2],
// K = [P + sigma I, A'; A, -diag(1/rho)], on the device: the counterpart of the reference's QdldlKKTSolver
// (kktsolver.jl:285-320).  The symbolic analysis (ordering, elimination tree, pattern of L, level schedules) runs on
// the host (ldl_symbolic.h); these kernels do everything numeric:
//
//   ldl_assemble_kernel   values of the permuted lower triangle of K from the resident P_, At_, rho_vec_ and sigma
//   ldl_factor_kernel     left-looking column LDL', one CTA per column, one launch per level (or per run of thin levels)
//   ldl_csr_gather_kernel the row-ordered copy of L the forward solve reads
//   ldl_forward_kernel    L z = P' r, one warp per row, the gather of the right-hand side fused in
//   ldl_backward_kernel   L' x = D^-1 z, one warp per column, the scatter into (y1, y2) fused in
//
// Every sum runs in a fixed order (columns k ascending in the factorisation, a fixed lane partition and shuffle tree
// in the solves) and nothing uses floating-point atomics, so a factorisation and a solve are bitwise reproducible.
// No CTA waits on another: levels are ordered by kernel boundaries, the levels of a run by __syncthreads() inside its
// single CTA.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "ldl_symbolic.h"

namespace cosmo {

// the sum of the sources of entry e of K, in the order the host listed them
template <typename T>
__device__ __forceinline__ T ldl_entry_value(int64_t e, const int64_t* __restrict__ Ksp, const int64_t* __restrict__ Ksrc,
                                             const T* __restrict__ Pval, const T* __restrict__ Atval,
                                             const T* __restrict__ rho, T sigma) {
  T v = T(0);
  for (int64_t s = Ksp[e]; s < Ksp[e + 1]; ++s) {
    const int64_t code = Ksrc[s];
    const int64_t idx = code >> 2;
    switch ((int)(code & 3)) {
      case ldl::SRC_P: v += Pval[idx]; break;
      case ldl::SRC_AT: v += Atval[idx]; break;
      case ldl::SRC_RHO: v += -T(1) / rho[idx]; break;
      default: v += sigma; break;
    }
  }
  return v;
}

template <typename T>
__global__ void ldl_assemble_kernel(int64_t nnz, const int64_t* __restrict__ Ksp, const int64_t* __restrict__ Ksrc,
                                    const T* __restrict__ Pval, const T* __restrict__ Atval, const T* __restrict__ rho,
                                    T sigma, T* __restrict__ Kx) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
    Kx[e] = ldl_entry_value(e, Ksp, Ksrc, Pval, Atval, rho, sigma);
}

template <typename T>
struct LdlFactorArgs {
  const int* cols;      // columns ordered by level
  const int* lptr;      // level pointers into cols
  int l0, l1;           // levels of this launch
  const int64_t* Kp; const int* Ki; const T* Kx;   // permuted lower triangle of K (diagonal first)
  const int64_t* Lp; const int* Li; T* Lx;        // L by columns
  const int64_t* Rp; const int* Rj; const int64_t* Rmap;   // L by rows, CSR -> CSC map
  T* D; T* Dinv;
  T* ws;                // gridDim.x dense workspaces of length N, zero between columns
  int64_t N;
  int* flags;           // [0] positive pivots, [1] zero or non-finite pivots
};

// Column j: w = K(j:N, j); w -= L(j:N, k) d_k L(j, k) for every k in row j of L (ascending); d_j = w_j;
// L(j+1:N, j) = w / d_j.  The entries of column k at rows >= j start at the CSC position of L(j, k) (rows ascending),
// so row j of L lists exactly where each update starts.  Only the rows of column j are touched and then cleared.
template <typename T>
__global__ void __launch_bounds__(kBlock) ldl_factor_kernel(LdlFactorArgs<T> a) {
  // (start, end, L(j,k) d_k) of up to kBlock updates, loaded in parallel: the sequential k loop then starts each update
  // from shared memory instead of a chain of dependent global loads
  __shared__ int64_t s_p[kBlock], s_end[kBlock];
  __shared__ T s_f[kBlock];
  T* w = a.ws + (int64_t)blockIdx.x * a.N;
  const int tid = threadIdx.x;
  for (int l = a.l0; l < a.l1; ++l) {
    for (int c = a.lptr[l] + blockIdx.x; c < a.lptr[l + 1]; c += gridDim.x) {
      const int j = a.cols[c];
      for (int64_t e = a.Kp[j] + tid; e < a.Kp[j + 1]; e += blockDim.x) w[a.Ki[e]] = a.Kx[e];
      const int64_t r1 = a.Rp[j + 1];
      for (int64_t r0 = a.Rp[j]; r0 < r1; r0 += kBlock) {
        if (r0 + tid < r1) {
          const int k = a.Rj[r0 + tid];
          const int64_t p = a.Rmap[r0 + tid];
          s_p[tid] = p;
          s_end[tid] = a.Lp[k + 1];
          s_f[tid] = a.Lx[p] * a.D[k];
        }
        __syncthreads();
        const int cnt = (int)min((int64_t)kBlock, r1 - r0);
        for (int t = 0; t < cnt; ++t) {
          const T f = s_f[t];
          const int64_t end = s_end[t];
          for (int64_t q = s_p[t] + tid; q < end; q += blockDim.x) w[a.Li[q]] -= a.Lx[q] * f;
          __syncthreads();
        }
      }
      __syncthreads();
      const T dj = w[j];
      const T inv = T(1) / dj;
      for (int64_t q = a.Lp[j] + tid; q < a.Lp[j + 1]; q += blockDim.x) {
        const int i = a.Li[q];
        a.Lx[q] = w[i] * inv;
        w[i] = T(0);
      }
      __syncthreads();
      if (tid == 0) {
        w[j] = T(0);
        a.D[j] = dj;
        a.Dinv[j] = inv;
        if (dj > T(0)) atomicAdd(a.flags, 1);
        if (!(dj != T(0)) || !isfinite(dj)) atomicAdd(a.flags + 1, 1);
      }
      __syncthreads();
    }
    __syncthreads();
  }
}

template <typename T>
__global__ void ldl_csr_gather_kernel(int64_t nnz, const int64_t* __restrict__ Rmap, const T* __restrict__ Lx, T* __restrict__ Rx) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nnz; r += (int64_t)gridDim.x * blockDim.x) Rx[r] = Lx[Rmap[r]];
}

__global__ void ldl_reset_flags_kernel(int* flags) {
  if (threadIdx.x < 2) flags[threadIdx.x] = 0;
}

template <typename T>
__device__ __forceinline__ T ldl_warp_sum(T s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

template <typename T>
struct LdlSolveArgs {
  const int* cols; const int* lptr; int l0, l1;
  const int64_t* ptr; const int* idx; const T* val;   // forward: L by rows; backward: L by columns
  const T* Dinv;
  const int* perm;
  const T* rhs;      // forward: [x1; x2] in the original order
  T* y;              // permuted work vector: z after the forward solve, x after the backward solve
  T* out1; T* out2;  // backward: y1 (n) and y2 (m) in the original order
  int n;
};

// z_i = rhs[perm[i]] - sum_k L(i, k) z_k
template <typename T>
__global__ void __launch_bounds__(kBlock) ldl_forward_kernel(LdlSolveArgs<T> a) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int l = a.l0; l < a.l1; ++l) {
    for (int c = a.lptr[l] + gw; c < a.lptr[l + 1]; c += nw) {
      const int i = a.cols[c];
      T s = T(0);
      for (int64_t r = a.ptr[i] + lane; r < a.ptr[i + 1]; r += 32) s += a.val[r] * a.y[a.idx[r]];
      s = ldl_warp_sum(s);
      if (lane == 0) a.y[i] = a.rhs[a.perm[i]] - s;
    }
    __syncthreads();
  }
}

// x_j = z_j / d_j - sum_{i > j} L(i, j) x_i, written in place of z_j and scattered to y1 / y2
template <typename T>
__global__ void __launch_bounds__(kBlock) ldl_backward_kernel(LdlSolveArgs<T> a) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int l = a.l0; l < a.l1; ++l) {
    for (int c = a.lptr[l] + gw; c < a.lptr[l + 1]; c += nw) {
      const int j = a.cols[c];
      T s = T(0);
      for (int64_t q = a.ptr[j] + lane; q < a.ptr[j + 1]; q += 32) s += a.val[q] * a.y[a.idx[q]];
      s = ldl_warp_sum(s);
      if (lane == 0) {
        const T x = a.y[j] * a.Dinv[j] - s;
        a.y[j] = x;
        const int o = a.perm[j];
        if (o < a.n) a.out1[o] = x;
        else a.out2[o - a.n] = x;
      }
    }
    __syncthreads();
  }
}

}  // namespace cosmo
