// adjoint.cuh -- derivatives of a polished QP or LP solution with respect to the data (cosmo_b200_adjoint, DESIGN.md §3j).
//
// After an accepted polish (polish.cuh) the engine holds the active set 𝒜, the polished point (x, nu) and, in the direct
// plugin's memory, the factor of the regularised K~ of that polish.  The adjoint of the solution map is one solve with
// the exact K_A = [P, A_A'; A_A, 0]:
//   K_A [u; v] = [D g_x - A' gs~; E g_y / c on A],   v = 0 off A,   gs~ = g_s / E
// in the engine's scaled coordinates, by the plugin's solves with that factor and iterative refinement against K_A (the
// polish's refinement passes with another right-hand side).  The kernels here form the right-hand side and turn (u, v)
// into the gradients of the unscaled data; each writes every output once, with no floating-point atomics, so a call is
// bitwise reproducible.  The gradients are formed in fp64 from the resident values of T.
#pragma once
#include "common.cuh"
#include "polish.cuh"

namespace cosmo {

// integer counters of the gradient pass (deterministic: integer atomics only)
enum { ADJ_CNT_ACTIVE = 0, ADJ_CNT_WEAK = 1, ADJ_CNT_COUNT = 2 };

// s rows of the right-hand side, one thread per row: gs~ = g_s / E, and r_s = E g_y / c on the active rows, 0 elsewhere,
// kept in rs and written into ls_ as the s rows of the first solve.  g_y, g_s null: zero.
template <typename T>
__global__ void __launch_bounds__(kBlock) adjoint_rhs_kernel(int n, int m, const unsigned char* __restrict__ kind,
                                                             const double* __restrict__ gy, const double* __restrict__ gs,
                                                             const T* __restrict__ E, double c, T* __restrict__ gs_t,
                                                             T* __restrict__ rs, T* __restrict__ ls) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const double e = E ? (double)E[r] : 1.0;
    gs_t[r] = gs ? (T)(gs[r] / e) : T(0);
    const T v = gy && kind[r] != POLISH_INACTIVE ? (T)(e * gy[r] / c) : T(0);
    rs[r] = v;
    ls[n + r] = v;
  }
}

// x rows of the right-hand side over A' gs~:  r_x = D g_x - A' gs~, kept in rx and written into ls_
template <typename T>
struct EpiAdjointRhsX {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* rx;
  T* ls;
  const double* gx;   // null: zero
  const T* D;         // null: identity
  __device__ void row(int j, T atg, T*, T*) const {
    const T d = gx ? (T)(D ? (double)D[j] * gx[j] : gx[j]) : T(0);
    const T v = d - atg;
    rx[j] = v;
    ls[j] = v;
  }
  __device__ void operator()(T*) const {}
};

template <typename T>
struct AdjointVecArgs {
  int n, m;
  const unsigned char* kind;        // POLISH_* of the polish
  const unsigned char* row_class;
  const T* u;                       // x part of the adjoint solution (n)
  const T* v;                       // s part, 0 off the active rows (m)
  const T* gs;                      // gs~ (m)
  const T* mu_p;                    // the polish's clipped multipliers (y = -mu_p)
  const T* D;                       // null: unscaled engine
  const T* E;
  double c;
  double* dq;                       // outputs, each may be null
  double* db;
  double* dl;
  double* du;
  int* counts;                      // ADJ_CNT_COUNT ints, zero on entry
};

// dq = -c D u,  db = E (v + gs~),  dl = -E v on lower-active Box rows,  du = -E v on upper-active ones, both -E v / 2 on
// Box rows with l = u, 0 elsewhere.  Counts the active rows and the inequality-active rows whose clipped multiplier is 0
// (weakly active: the derivative there is one-sided).  One thread per entry of [x; s].
template <typename T>
__global__ void __launch_bounds__(kBlock) adjoint_grad_vec_kernel(AdjointVecArgs<T> a) {
  const int total = a.n + a.m;
  const int stride = gridDim.x * blockDim.x;
  // every thread of the block runs the same number of rounds (__syncthreads_count below)
  const int rounds = (total + stride - 1) / stride;
  for (int k = 0, idx = blockIdx.x * blockDim.x + threadIdx.x; k < rounds; ++k, idx += stride) {
    bool active = false, weak = false;
    if (idx < a.n) {
      if (a.dq) a.dq[idx] = -(a.D ? a.c * (double)a.D[idx] : a.c) * (double)a.u[idx];
    } else if (idx < total) {
      const int r = idx - a.n;
      const unsigned char kd = a.kind[r];
      const double e = a.E ? (double)a.E[r] : 1.0;
      const double v = (double)a.v[r];
      if (a.db) a.db[r] = e * (v + (double)a.gs[r]);
      double lo = 0.0, up = 0.0;
      if (a.row_class[r] == ROW_BOX) {
        if (kd == POLISH_LOWER) lo = -e * v;
        else if (kd == POLISH_UPPER) up = -e * v;
        else if (kd == POLISH_EQUALITY) lo = up = -0.5 * (e * v);
      }
      if (a.dl) a.dl[r] = lo;
      if (a.du) a.du[r] = up;
      active = kd != POLISH_INACTIVE;
      weak = (kd == POLISH_LOWER || kd == POLISH_UPPER) && a.mu_p[r] == T(0);
    }
    const int na = __syncthreads_count(active);
    const int nw = __syncthreads_count(weak);
    if (threadIdx.x == 0) {
      if (na) atomicAdd(a.counts + ADJ_CNT_ACTIVE, na);
      if (nw) atomicAdd(a.counts + ADJ_CNT_WEAK, nw);
    }
  }
}

// dP over CSR(P), one warp per row: dP_ij = -c D_i D_j (u_i x_j + x_i u_j) / 2, written at the caller's CSC index src[k].
// The formula is symmetric bit for bit in (i, j), so both stored triangles get the same value.
template <typename T>
__global__ void __launch_bounds__(kBlock) adjoint_grad_P_kernel(int n, const int* __restrict__ rowptr, const int* __restrict__ col,
                                                                const int* __restrict__ src, const T* __restrict__ u,
                                                                const T* __restrict__ x, const T* __restrict__ D, double c,
                                                                double* __restrict__ dPx) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const double ui = (double)u[i], xi = (double)x[i], di = D ? (double)D[i] : 1.0;
    for (int k = rowptr[i] + lane; k < rowptr[i + 1]; k += 32) {
      const int j = col[k];
      const double dj = D ? (double)D[j] : 1.0;
      dPx[src[k]] = -(c * (di * dj)) * (0.5 * (ui * (double)x[j] + xi * (double)u[j]));
    }
  }
}

// dA over CSR(A') (its value order is A's CSC order), one warp per column j of A:
//   dA_rj = E_r D_j (-(y_r u_j + v_r x_j) - gs~_r x_j),   y = -mu_p  (gs null: no gs~ term; the solve adjoint)
template <typename T>
__global__ void __launch_bounds__(kBlock) adjoint_grad_A_kernel(int n, const int* __restrict__ rowptr, const int* __restrict__ col,
                                                                const T* __restrict__ u, const T* __restrict__ x,
                                                                const T* __restrict__ v, const T* __restrict__ mu_p,
                                                                const T* __restrict__ gs, const T* __restrict__ D,
                                                                const T* __restrict__ E, double* __restrict__ dAx) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += warps) {
    const double uj = (double)u[j], xj = (double)x[j], dj = D ? (double)D[j] : 1.0;
    for (int k = rowptr[j] + lane; k < rowptr[j + 1]; k += 32) {
      const int r = col[k];
      const double y = -(double)mu_p[r];
      const double g = -(y * uj + (double)v[r] * xj) - (gs ? (double)gs[r] * xj : 0.0);
      dAx[k] = (E ? (double)E[r] * dj : dj) * g;
    }
  }
}

// out[0 .. count) = NaN: the outputs of a call whose status is not 1
__global__ void __launch_bounds__(kBlock) adjoint_nan_kernel(long long count, double* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
    out[i] = __longlong_as_double(0x7ff8000000000000LL);
}

}  // namespace cosmo
