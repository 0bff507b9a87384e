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

// Adds the block's active rows and its weakly active ones (lower- or upper-active rows whose clipped multiplier is 0:
// the derivative there is one-sided) to counts, for row r of the polish (r outside 0 .. m: none).  Every thread of the
// block calls it once per round (__syncthreads_count).
template <typename T>
__device__ __forceinline__ void adj_count_rows(int r, int m, const unsigned char* __restrict__ kind,
                                               const T* __restrict__ mu_p, int* __restrict__ counts) {
  bool active = false, weak = false;
  if (r >= 0 && r < m) {
    const unsigned char kd = kind[r];
    active = kd != POLISH_INACTIVE;
    weak = (kd == POLISH_LOWER || kd == POLISH_UPPER) && mu_p[r] == T(0);
  }
  const int na = __syncthreads_count(active);
  const int nw = __syncthreads_count(weak);
  if (threadIdx.x == 0) {
    if (na) atomicAdd(counts + ADJ_CNT_ACTIVE, na);
    if (nw) atomicAdd(counts + ADJ_CNT_WEAK, nw);
  }
}

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
    }
    adj_count_rows(idx - a.n, a.m, a.kind, a.mu_p, a.counts);
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

// ---- the forward derivative (cosmo_b200_derivative, DESIGN.md §3j) -----------------------------------------------
// The transpose of the adjoint above, with the same K_A, factor and refinement:
//   K_A [x'; y'_A] = [-dq~ - dP~ x~ - dA~' y~; e - sbar'~ on A],   y' = 0 off A,   e = E db - dA~ x~,   s~' = e - A~ x'.
// The x rows are sd_rhs_x_kernel's (solve_adjoint.cuh) at the polished point, s~' is one SpMV pass with
// EpiPolishSlack; the two kernels below form the s rows and write the outputs.

// s rows of the right-hand side, one warp per CSR(A) row r (map: CSR position -> CSC index of A's values):
//   e_r = E_r db_r - (dA~ x~)_r on every row, kept in e for s~',
//   r_s = e_r - sbar'_r on the active rows, 0 elsewhere, kept in rs and written into ls_s for the first solve,
// with sbar' the scaled bound direction: E dl on lower-active Box rows, E du on upper-active ones, E (dl + du) / 2 on
// Box rows with l = u (the transpose of adjoint_grad_vec_kernel's half split), 0 on ZeroSet and Nonnegatives rows.
// dAx, db, dl, du null: zero.
template <typename T>
__global__ void __launch_bounds__(kBlock) derivative_rhs_s_kernel(int m, const int* __restrict__ a_rowptr, const int* __restrict__ a_col,
                                                                  const int* __restrict__ map, const double* __restrict__ dAx,
                                                                  const double* __restrict__ db, const double* __restrict__ dl,
                                                                  const double* __restrict__ du, const unsigned char* __restrict__ kind,
                                                                  const unsigned char* __restrict__ row_class,
                                                                  const T* __restrict__ x, const T* __restrict__ D,
                                                                  const T* __restrict__ E, T* __restrict__ e_out,
                                                                  T* __restrict__ rs, T* __restrict__ ls_s) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < m; r += warps) {
    const double e = E ? (double)E[r] : 1.0;
    double acc = 0.0;
    if (dAx)
      for (int k = a_rowptr[r] + lane; k < a_rowptr[r + 1]; k += 32) {
        const int j = a_col[k];
        acc += e * (D ? (double)D[j] : 1.0) * dAx[map[k]] * (double)x[j];
      }
    acc = warp_sum(acc);
    if (lane == 0) {
      const double er = (db ? e * db[r] : 0.0) - acc;
      const unsigned char kd = kind[r];
      double sb = 0.0;
      if (row_class[r] == ROW_BOX) {
        const double lo = dl ? e * dl[r] : 0.0, up = du ? e * du[r] : 0.0;
        if (kd == POLISH_LOWER) sb = lo;
        else if (kd == POLISH_UPPER) sb = up;
        else if (kd == POLISH_EQUALITY) sb = 0.5 * (lo + up);
      }
      const T v = kd != POLISH_INACTIVE ? (T)(er - sb) : T(0);
      e_out[r] = (T)er;
      rs[r] = v;
      ls_s[r] = v;
    }
  }
}

// the outputs, unscaled as cosmo_b200_solution unscales the solution: dx = D x~',  dy = E y~' / c on the active rows
// and 0 elsewhere,  ds = s~' / E; counts the rows as adjoint_grad_vec_kernel does.  One thread per entry of [x; s].
template <typename T>
__global__ void __launch_bounds__(kBlock) derivative_out_kernel(int n, int m, const unsigned char* __restrict__ kind,
                                                                const T* __restrict__ mu_p, const T* __restrict__ xd,
                                                                const T* __restrict__ yd, const T* __restrict__ sd,
                                                                const T* __restrict__ D, const T* __restrict__ E, double c,
                                                                double* __restrict__ dx, double* __restrict__ dy,
                                                                double* __restrict__ ds, int* __restrict__ counts) {
  const int total = n + m;
  // the loop bound is the block's first index, so every thread of the block runs the same rounds (adj_count_rows)
  for (int first = blockIdx.x * blockDim.x; first < total; first += gridDim.x * blockDim.x) {
    const int idx = first + threadIdx.x;
    if (idx < n) {
      if (dx) dx[idx] = (D ? (double)D[idx] : 1.0) * (double)xd[idx];
    } else if (idx < total) {
      const int r = idx - n;
      const double e = E ? (double)E[r] : 1.0;
      if (dy) dy[r] = kind[r] != POLISH_INACTIVE ? e * (double)yd[r] / c : 0.0;
      if (ds) ds[r] = (double)sd[r] / e;
    }
    adj_count_rows(idx - n, m, kind, mu_p, counts);
  }
}

// out[0 .. count) = NaN: the outputs of a call whose status is not 1
__global__ void __launch_bounds__(kBlock) adjoint_nan_kernel(long long count, double* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
    out[i] = __longlong_as_double(0x7ff8000000000000LL);
}

}  // namespace cosmo
