// polish.cuh -- solution polishing of QPs and LPs (cosmo_b200_polish, DESIGN.md §3i).
//
// From the resident ADMM solution (x, s, mu) the engine guesses the active rows, solves the equality-constrained KKT
// system of that guess through the direct LDL' plugin (regularised, then iteratively refined) and keeps the result only
// if its residuals are no worse.  The kernels here are the elementwise steps of that procedure; the products go through
// the engine's SpMV passes (the epilogues below), the factor and the solves through the plugin, the slack through the
// projection of proj_rhs_kernel and the residuals through compute_residuals.
//
// Unknown z = (x, nu) with nu = -mu.  The plugin factors K~ = [P + sigma I, A'; A, -diag(1 / rho)]; polishing sets
// sigma = delta, rho = 1 / delta on the active rows and rho = delta elsewhere.  The exact reduced system, embedded in
// n + m rows, is
//   P x + A' nu = -q,   (A x)_i = b_i - sbar_i on active rows,   nu_i = 0 on the others.
#pragma once
#include "common.cuh"
#include "vector_kernels.cuh"

namespace cosmo {

// active kind of a row
enum : unsigned char { POLISH_INACTIVE = 0, POLISH_LOWER = 1, POLISH_UPPER = 2, POLISH_EQUALITY = 3 };
// integer counters of the classification (deterministic: integer atomics only)
enum { POLISH_CNT_LOWER = 0, POLISH_CNT_UPPER = 1, POLISH_CNT_EQ = 2, POLISH_CNT_COUNT = 4 };

template <typename T>
struct PolishClassifyArgs {
  int n, m;
  const unsigned char* row_class;
  const T* box_l;
  const T* box_u;
  const T* b;
  const T* q;
  const T* s;            // resident slack
  const T* mu;           // resident mu (y = -mu)
  T delta;
  unsigned char* kind;   // out: POLISH_*
  T* rhs;                // out: b - sbar on active rows, 0 elsewhere (m)
  T* rho;                // out: the polish rho vector (m)
  const T* x;            // resident x
  T* ls;                 // out: the first right-hand side [-q + delta x; rhs + delta mu on the active rows] (n + m)
  int* counts;           // POLISH_CNT_COUNT ints, zero on entry
  T* nq;                 // out: -q, the x rows of the exact right-hand side (n)
};

// Row classification (DESIGN §3i step 1) and the first right-hand side, one thread per entry of [x; s].  The first
// solve is centred at the ADMM iterate z0 = (x, -mu on the active rows): K~ z1 = r^ + (K~ - K_A) z0, i.e. the first
// refinement step from z0 with its residual formed elementwise.  Where the active rows are linearly dependent (an
// equality written as two inequalities) the multipliers are not unique, and z0 keeps the split ADMM found, which lies in
// the normal cone, instead of the minimum-norm split of the regularised solve.
//   equality:  ZeroSet rows, Box rows with l = u                     sbar = 0, l
//   lower:     Nonnegatives with s < -mu;  Box with s - l < -mu       sbar = 0, l
//   upper:     Box with u - s < mu (when not lower)                   sbar = u
// An infinite bound gives an infinite gap and is never active; NaN compares false.
template <typename T>
__global__ void __launch_bounds__(kBlock) polish_classify_kernel(PolishClassifyArgs<T> a) {
  const int total = a.n + a.m;
  const int stride = gridDim.x * blockDim.x;
  // every thread of the block runs the same number of rounds (__syncthreads_count below)
  const int rounds = (total + stride - 1) / stride;
  for (int k = 0, idx = blockIdx.x * blockDim.x + threadIdx.x; k < rounds; ++k, idx += stride) {
    unsigned char kd = POLISH_INACTIVE;
    if (idx < a.n) {
      a.ls[idx] = a.delta * a.x[idx] - a.q[idx];
      a.nq[idx] = -a.q[idx];
    } else if (idx < total) {
      const int r = idx - a.n;
      const unsigned char cls = a.row_class[r];
      const T sr = a.s[r], mr = a.mu[r];
      T sbar = T(0);
      if (cls == ROW_ZERO) {
        kd = POLISH_EQUALITY;
      } else if (cls == ROW_NONNEG) {
        if (sr < -mr) kd = POLISH_LOWER;
      } else if (cls == ROW_BOX) {
        const T l = a.box_l[r], u = a.box_u[r];
        if (l == u) { kd = POLISH_EQUALITY; sbar = l; }
        else if (sr - l < -mr) { kd = POLISH_LOWER; sbar = l; }
        else if (u - sr < mr) { kd = POLISH_UPPER; sbar = u; }
      }
      const T rh = kd != POLISH_INACTIVE ? a.b[r] - sbar : T(0);
      a.kind[r] = kd;
      a.rhs[r] = rh;
      a.ls[idx] = kd != POLISH_INACTIVE ? rh + a.delta * mr : T(0);
      a.rho[r] = kd != POLISH_INACTIVE ? T(1) / a.delta : a.delta;
    }
    const int nl = __syncthreads_count(kd == POLISH_LOWER);
    const int nu = __syncthreads_count(kd == POLISH_UPPER);
    const int ne = __syncthreads_count(kd == POLISH_EQUALITY);
    if (threadIdx.x == 0) {
      if (nl) atomicAdd(a.counts + POLISH_CNT_LOWER, nl);
      if (nu) atomicAdd(a.counts + POLISH_CNT_UPPER, nu);
      if (ne) atomicAdd(a.counts + POLISH_CNT_EQ, ne);
    }
  }
}

// z <- dz (first) or z + dz, with nu_i = 0 off the active rows (DESIGN §3i step 4); dz = [xsol; nu] of the plugin
template <typename T>
__global__ void __launch_bounds__(kBlock) polish_update_kernel(int n, int m, const unsigned char* __restrict__ kind,
                                                               const T* __restrict__ dx, const T* __restrict__ dnu,
                                                               T* __restrict__ zx, T* __restrict__ znu, int first) {
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n + m; idx += gridDim.x * blockDim.x) {
    if (idx < n) {
      zx[idx] = first ? dx[idx] : zx[idx] + dx[idx];
    } else {
      const int r = idx - n;
      znu[r] = kind[r] == POLISH_INACTIVE ? T(0) : (first ? dnu[r] : znu[r] + dnu[r]);
    }
  }
}

// mu_p = -nu on the active rows, clipped into the normal cone of the row's set at sbar (<= 0 at a lower bound, >= 0 at
// an upper bound, free on an equality row), 0 elsewhere (DESIGN §3i step 5)
template <typename T>
__global__ void __launch_bounds__(kBlock) polish_finish_kernel(int m, const unsigned char* __restrict__ kind,
                                                               const T* __restrict__ nu, T* __restrict__ mu_p) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const unsigned char kd = kind[r];
    const T v = -nu[r];
    T out = T(0);
    if (kd == POLISH_EQUALITY) out = v;
    else if (kd == POLISH_LOWER) out = v < T(0) ? v : T(0);
    else if (kd == POLISH_UPPER) out = v > T(0) ? v : T(0);
    mu_p[r] = out;
  }
}

// ---- SpMV epilogues of the refinement residual and the candidate slack --------------------------------------------
// x rows of r^ - K_A z over A' nu (px = P x precomputed):  r_x = rx - P x - A' nu,   max0 = |r_x|_inf.  rx is -q for the
// polish (the negation is exact, so this is -q - P x - A' nu bit for bit) and the adjoint's right-hand side for
// cosmo_b200_adjoint (adjoint.cuh).
template <typename T>
struct EpiPolishResX {
  static constexpr int NS = 0, NM = 1;
  const int* done;
  T* out;
  const T* rx;
  const T* px;
  __device__ void row(int r, T atnu, T*, T* accM) const {
    const T v = rx[r] - (px[r] + atnu);
    out[r] = v;
    accM[0] = nanmax(accM[0], tabs(v));
  }
  __device__ void operator()(T*) const {}
};

// s rows over A x:  r_s = rhs - A x on the active rows, 0 elsewhere,   max0 = |r_s|_inf (rhs: b - sbar for the polish,
// the adjoint's s rows for cosmo_b200_adjoint)
template <typename T>
struct EpiPolishResS {
  static constexpr int NS = 0, NM = 1;
  const int* done;
  T* out;
  const T* rhs;
  const unsigned char* kind;
  __device__ void row(int r, T ax, T*, T* accM) const {
    const T v = kind[r] != POLISH_INACTIVE ? rhs[r] - ax : T(0);
    out[r] = v;
    accM[0] = nanmax(accM[0], tabs(v));
  }
  __device__ void operator()(T*) const {}
};

// w_s = b - A x: the argument of the slack projection s_p = Pi_K(b - A x_p)
template <typename T>
struct EpiPolishSlack {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* ws;
  const T* b;
  __device__ void row(int r, T ax, T*, T*) const { ws[r] = b[r] - ax; }
  __device__ void operator()(T*) const {}
};

}  // namespace cosmo
