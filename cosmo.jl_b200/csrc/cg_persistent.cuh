// cg_persistent.cuh -- the whole reduced-KKT CG solve in ONE cooperative launch.
//
// For small / medium problems the CG inner loop of kktsolver_indirect.jl:70 is bound by launch
// latency, not by HBM: every iteration is five microsecond-sized kernels.  This kernel keeps one
// grid resident (<= one CTA wave) and walks the iterations itself; the phases of an iteration are
// separated by grid-wide barriers (cooperative groups), the scalars (alpha, beta, residual norm,
// tolerance test) are recomputed redundantly by every block from per-block partials folded in a fixed
// order -- deterministic, and no host round trip: the host never waits for the inner solver, so an
// entire ADMM iteration is enqueued without a single synchronisation.
//
//   rhs given;  x = warm start (previous solution)
//   c = L x ; r = rhs - c ; u = 0 ; res = |r| ; tol = tol_num / |rhs|
//   while res > tol and it < maxit:
//       u = r + (res/prev)^2 u ; c = L u ; alpha = res^2 / u'c ; x += alpha u ; r -= alpha c
// with  L v = A'(rho .* (A v)) + P v + sigma v   (reduced_mul!, kktsolver_indirect.jl:57-67).
#pragma once
#include <cooperative_groups.h>

#include "spmv.cuh"
#include "vector_kernels.cuh"

namespace cosmo {

template <typename T>
struct CgPersistArgs {
  CsrView<T> A, At, P;
  int n, m;
  const T* rhs;
  const T* rho;
  T* x;
  T* r;
  T* u;
  T* tm;      // m
  T* c;       // n
  T* partA;   // gridDim * 2
  T* partB;   // gridDim * 2
  T* sc;
  int* isc;   // [ISC_DONE], [ISC_IT], [ISC_MAXIT], [ISC_TOTAL] accumulates inner iterations
  T sigma;
  T tol_num;
};

enum { ISC_TOTAL = 4 };

// block partial of up to two sums -> part[blockIdx * 2 + k]
template <typename T>
__device__ __forceinline__ void block_partials2(T a0, T a1, T* part) {
  __shared__ T sm[kWarpsPerBlock][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  if (lane == 0) { sm[warp][0] = a0; sm[warp][1] = a1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    T s0 = sm[0][0], s1 = sm[0][1];
    for (int w = 1; w < kWarpsPerBlock; ++w) { s0 += sm[w][0]; s1 += sm[w][1]; }
    part[blockIdx.x * 2] = s0;
    part[blockIdx.x * 2 + 1] = s1;
  }
  __syncthreads();
}

// every block folds all partials in the same fixed order (after a grid barrier)
template <typename T>
__device__ __forceinline__ void fold_partials2(const T* part, T& s0, T& s1) {
  __shared__ T res[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp == 0) {
    T a0 = 0, a1 = 0;
    for (int b = lane; b < (int)gridDim.x; b += 32) {
      a0 += __ldcg(part + b * 2);
      a1 += __ldcg(part + b * 2 + 1);
    }
    a0 = warp_sum(a0);
    a1 = warp_sum(a1);
    if (lane == 0) { res[0] = a0; res[1] = a1; }
  }
  __syncthreads();
  s0 = res[0];
  s1 = res[1];
  __syncthreads();
}

template <typename T, int LANES>
__global__ void __launch_bounds__(kBlock) cg_persistent_kernel(CgPersistArgs<T> a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  constexpr int GROUPS = kBlock / LANES;
  const int lane = threadIdx.x % LANES, group = threadIdx.x / LANES;
  const int total_groups = gridDim.x * GROUPS;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
  const int maxit = a.isc[ISC_MAXIT];

  // tm = rho .* (A v)
  auto stage1 = [&](const T* v) {
    for (int base = blockIdx.x * GROUPS; base < a.m; base += total_groups) {
      const int row = base + group;
      T s = 0;
      if (row < a.m) s = row_partial<T, LANES, false>(a.A, v, row, lane);
      s = group_sum<T, LANES>(s);
      if (row < a.m && lane == 0) a.tm[row] = a.rho[row] * s;
    }
  };
  // c_i = (A' tm)_i + (P v)_i + sigma v_i ; calls f(i, c_i) on the owning lane
  auto stage2 = [&](const T* v, auto&& f) {
    for (int base = blockIdx.x * GROUPS; base < a.n; base += total_groups) {
      const int row = base + group;
      T s = 0;
      if (row < a.n) {
        s = row_partial<T, LANES, false>(a.At, a.tm, row, lane);
        s += row_partial<T, LANES, false>(a.P, v, row, lane);
      }
      s = group_sum<T, LANES>(s);
      if (row < a.n && lane == 0) f(row, s + a.sigma * __ldcg(v + row));
    }
  };

  // ---- initial residual (warm start: one product) ----
  stage1(a.x);
  grid.sync();
  T acc0 = 0, acc1 = 0;
  stage2(a.x, [&](int i, T ci) {
    const T b = a.rhs[i];
    const T ri = b - ci;
    a.r[i] = ri;
    a.u[i] = T(0);
    acc0 += ri * ri;
    acc1 += b * b;
  });
  block_partials2(acc0, acc1, a.partA);
  grid.sync();
  T res2, rhs2;
  fold_partials2(a.partA, res2, rhs2);
  T res = sqrt(res2), prev = T(1);
  const T tol = inner_abstol(a.tol_num, sqrt(rhs2));
  int it = 0;

  while (!(res <= tol) && it < maxit) {
    const T beta = (res * res) / (prev * prev);
    for (int i = tid; i < a.n; i += nthreads) a.u[i] = __ldcg(a.r + i) + beta * __ldcg(a.u + i);
    grid.sync();
    stage1(a.u);
    grid.sync();
    acc0 = 0;
    stage2(a.u, [&](int i, T ci) {
      a.c[i] = ci;
      acc0 += __ldcg(a.u + i) * ci;
    });
    block_partials2(acc0, T(0), a.partB);
    grid.sync();
    T dot, dummy;
    fold_partials2(a.partB, dot, dummy);
    const T alpha = (res * res) / dot;
    acc0 = 0;
    for (int i = tid; i < a.n; i += nthreads) {
      a.x[i] = __ldcg(a.x + i) + alpha * __ldcg(a.u + i);
      const T ri = __ldcg(a.r + i) - alpha * __ldcg(a.c + i);
      a.r[i] = ri;
      acc0 += ri * ri;
    }
    block_partials2(acc0, T(0), a.partA);
    grid.sync();
    fold_partials2(a.partA, res2, dummy);
    prev = res;
    res = sqrt(res2);
    ++it;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.sc[SC_RES] = res;
    a.sc[SC_PREV] = prev;
    a.sc[SC_TOL] = tol;
    a.isc[ISC_IT] = it;
    a.isc[ISC_DONE] = 1;
    a.isc[ISC_TOTAL] += it;
  }
}

}  // namespace cosmo
