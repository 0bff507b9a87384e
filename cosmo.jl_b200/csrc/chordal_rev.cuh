// chordal_rev.cuh -- the reverse of a chordal decomposition on the device: reverse_scaling! + reverse_decomposition!
// + psd_completion! (scaling.jl:170-179, chordal_decomposition.jl:129-311).
//
// The map is computed once on the host (chordal.decomposition_arrays) and handed over with
// cosmo_b200_set_decomposition (compact transformation) or cosmo_b200_set_decomposition_noncompact (the traditional
// one, s = H s', chordal_decomposition.jl:136-168).  One reverse is:
//   1. gather_kernel: x = D x'[:n_orig]; for every original row of a decomposed cone s = 0.0 + the sum of its clique
//      rows in the host's order; mu = the last of them (compact) or (0.0 + the same sum over mu') / their count
//      (traditional: H mu' divided by the row's overlap count).  Plain rows are copied (compact) or are 0.0 + the
//      row (traditional: they are rows of H s' too).  One thread per output entry, no atomics: the result is
//      bit-identical to chordal.reverse on the same fp64 inputs.
//   2. with complete_dual, per decomposed cone (psd_complete, chordal_decomposition.jl:262-311):
//      a. scatter_kernel: W = mat(-mu) in the traversal numbering (dense, column-major, N x N); a square PsdCone is
//         read from its upper triangle (Symmetric(mat(-mu), :U)).
//      b. solve_kernel, one CTA per clique: Z = W[alpha, alpha] \ W[alpha, nu] in shared memory (Cholesky; LU with
//         partial pivoting where it fails; the pseudo-inverse through a Jacobi eigendecomposition where the LU pivot
//         is exactly zero or Z is not finite, as numpy.linalg.solve / pinv).  Both blocks lie inside the clique, and the
//         completion never changes an entry inside a clique, so every Z can be formed before the first update.
//      c. update_kernel, one cooperative launch: the cliques in traversal order, a grid barrier between two of them
//         (clique t reads W[:lo, alpha], which the cliques before it filled); W[r, nu] = W[nu, r] = W[r, alpha] Z for the
//         rows r < lo outside the clique.
//      d. gather_back_kernel: mu = -svec(W) over the cone's rows (all N^2 entries of a square cone).
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <iterator>
#include <string>
#include <utility>
#include <vector>

#include "../../include/cosmo_b200.h"
#include "host.cuh"

namespace cosmo {
namespace rev {

constexpr double kSqrt2 = 0x1.6a09e667f3bcdp+0;      // np.sqrt(2.0)
constexpr double kInvSqrt2 = 0x1.6a09e667f3bccp-1;   // 1.0 / np.sqrt(2.0), as _svec_to_mat scales
constexpr double kPinvRcond = 1e-15;                  // numpy.linalg.pinv: singular values <= 1e-15 * max are dropped
constexpr int kThreads = 256;
constexpr int kSolveThreads = 128;
constexpr int kJacobiSweeps = 60;
constexpr size_t kMaxSmem = 227 * 1024;

// (i, j), i <= j, of position k of the column-major upper triangle
__device__ __forceinline__ void svec_ij(int64_t k, int64_t& i, int64_t& j) {
  int64_t jj = (int64_t)((sqrt(8.0 * (double)k + 1.0) - 1.0) * 0.5);
  while ((jj + 1) * (jj + 2) / 2 <= k) ++jj;
  while (jj * (jj + 1) / 2 > k) --jj;
  j = jj;
  i = k - jj * (jj + 1) / 2;
}

template <typename T>
struct GatherArgs {
  int64_t n_orig, n_rows, n_plain, plain_rows;
  const T* x;                 // the engine's iterates, scaled
  const T* s;
  const T* mu;
  const T* D;                 // NULL: identity scaling
  const T* E;
  double c;
  const int64_t* row;
  const int64_t* s_ptr;
  const int64_t* s_src;
  const int64_t* mu_src;
  const int64_t* plain;       // 3 per block
  const int64_t* plain_pref;  // n_plain + 1
  int traditional;            // mu is the mean over s_src (mu_src unused); plain rows are 0.0 + the row
  double* x_out;              // NULL: skipped
  double* s_out;
  double* mu_out;
};

// reverse_scaling! of one row, widened to fp64 first as the host does: s / E and (E mu) / c
template <typename T>
__device__ __forceinline__ double unscale_s(const GatherArgs<T>& a, int64_t r) {
  return (double)a.s[r] / (a.E ? (double)a.E[r] : 1.0);
}
template <typename T>
__device__ __forceinline__ double unscale_mu(const GatherArgs<T>& a, int64_t r) {
  return ((a.E ? (double)a.E[r] : 1.0) * (double)a.mu[r]) / a.c;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) gather_kernel(GatherArgs<T> a) {
  const int64_t total = a.n_orig + a.n_rows + a.plain_rows;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    if (t < a.n_orig) {
      if (a.x_out) a.x_out[t] = (a.D ? (double)a.D[t] : 1.0) * (double)a.x[t];
    } else if (t < a.n_orig + a.n_rows) {
      const int64_t i = t - a.n_orig, r = a.row[i];
      if (a.s_out) {
        double acc = 0.0;
        for (int64_t p = a.s_ptr[i]; p < a.s_ptr[i + 1]; ++p) acc += unscale_s(a, a.s_src[p]);
        a.s_out[r] = acc;
      }
      if (a.mu_out && a.traditional) {
        double acc = 0.0;
        for (int64_t p = a.s_ptr[i]; p < a.s_ptr[i + 1]; ++p) acc += unscale_mu(a, a.s_src[p]);
        const int64_t cnt = a.s_ptr[i + 1] - a.s_ptr[i];
        a.mu_out[r] = cnt > 1 ? acc / (double)cnt : acc;
      } else if (a.mu_out) {
        a.mu_out[r] = unscale_mu(a, a.mu_src[i]);
      }
    } else {
      const int64_t q = t - a.n_orig - a.n_rows;
      int64_t lo = 0, hi = a.n_plain - 1;            // the last block that starts at or before q
      while (lo < hi) {
        const int64_t mid = (lo + hi + 1) / 2;
        if (a.plain_pref[mid] <= q) lo = mid; else hi = mid - 1;
      }
      const int64_t k = q - a.plain_pref[lo], old = a.plain[3 * lo] + k, nw = a.plain[3 * lo + 1] + k;
      if (a.s_out) {                                  // 0.0 + v: a -0.0 arrives as +0.0, as H s' gives it
        const double v = unscale_s(a, nw);
        a.s_out[old] = a.traditional ? 0.0 + v : v;
      }
      if (a.mu_out) {
        const double v = unscale_mu(a, nw);
        a.mu_out[old] = a.traditional ? 0.0 + v : v;
      }
    }
  }
}

// W = mat(-v) in the traversal numbering (_svec_to_mat: off-diagonal entries (y + 0) / sqrt 2).  A square cone
// (column-major N x N) is read from its upper triangle, every entry y + 0 as np.triu(Y) + np.triu(Y, 1).T gives it.
__global__ void __launch_bounds__(kThreads) scatter_kernel(int64_t N, const double* v, const int64_t* new_of, double* W,
                                                           int square) {
  const int64_t dim = N * (N + 1) / 2;
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < dim; k += (int64_t)gridDim.x * blockDim.x) {
    int64_t i, j;
    svec_ij(k, i, j);
    const double y = -v[square ? i + N * j : k];
    const int64_t ni = new_of[i], nj = new_of[j];
    if (square) {
      W[ni + N * nj] = y + 0.0;
      W[nj + N * ni] = y + 0.0;
    } else if (i == j) {
      W[ni + N * ni] = y;
    } else {
      const double w = (y + 0.0) * kInvSqrt2;
      W[ni + N * nj] = w;
      W[nj + N * ni] = w;
    }
  }
}

// v = -svec(W) (_mat_to_svec: off-diagonal entries times sqrt 2); v = -vec(W) over all N^2 entries of a square cone
__global__ void __launch_bounds__(kThreads) gather_back_kernel(int64_t N, const int64_t* new_of, const double* W, double* v,
                                                               int square) {
  const int64_t dim = square ? N * N : N * (N + 1) / 2;
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < dim; k += (int64_t)gridDim.x * blockDim.x) {
    if (square) {
      v[k] = -W[new_of[k % N] + N * new_of[k / N]];
      continue;
    }
    int64_t i, j;
    svec_ij(k, i, j);
    const double y = W[new_of[j] + N * new_of[i]];
    v[k] = i == j ? -y : -(y * kSqrt2);
  }
}

// y = -mu of the reversed solution (cosmo_b200_solution)
__global__ void __launch_bounds__(kThreads) negate_kernel(int64_t n, double* v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) v[i] = -v[i];
}

// the bare matrix of cosmo_b200_psd_complete: its upper triangle into the traversal numbering, and back
__global__ void __launch_bounds__(kThreads) permute_in_kernel(int64_t N, const double* Y, const int64_t* new_of, double* W) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N * N; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e % N, j = e / N;
    W[new_of[i] + N * new_of[j]] = i <= j ? Y[i + N * j] : Y[j + N * i];
  }
}
__global__ void __launch_bounds__(kThreads) permute_out_kernel(int64_t N, const double* W, const int64_t* new_of, double* Y) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N * N; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e % N, j = e / N;
    Y[e] = W[new_of[i] + N * new_of[j]];
  }
}

struct StepTable {
  int64_t n_steps;
  const int64_t* steps;   // 6 per step: lo, hi, a0, a1, k0, k1
  const int64_t* idx;
  const int64_t* z_off;   // n_steps: start of the step's Z (|alpha| x |nu|, column-major) in the Z buffer
};

// ---- small dense solves of one CTA in shared memory (column-major a x a) ----------------------------------------
__device__ bool block_cholesky(double* F, int a, int* flag) {
  for (int k = 0; k < a; ++k) {
    if (threadIdx.x == 0) {
      const double d = F[k + a * k];
      *flag = (d > 0.0 && isfinite(d)) ? 0 : 1;
      if (!*flag) F[k + a * k] = sqrt(d);
    }
    __syncthreads();
    if (*flag) return false;
    const double dk = F[k + a * k];
    for (int i = k + 1 + threadIdx.x; i < a; i += blockDim.x) F[i + a * k] /= dk;
    __syncthreads();
    const int r = a - k - 1;
    for (int e = threadIdx.x; e < r * r; e += blockDim.x) {
      const int i = k + 1 + e % r, j = k + 1 + e / r;
      if (j <= i) F[i + a * j] -= F[i + a * k] * F[j + a * k];
    }
    __syncthreads();
  }
  return true;
}

// LU with partial pivoting (dgetrf's choice: the first entry of largest magnitude); the row swaps are applied to X too.
// False when a pivot is exactly zero (dgesv's info > 0: numpy raises LinAlgError).
__device__ bool block_lu(double* F, double* X, int a, int nn, int* flag) {
  for (int k = 0; k < a; ++k) {
    if (threadIdx.x == 0) {
      int p = k;
      double best = fabs(F[k + a * k]);
      for (int i = k + 1; i < a; ++i)
        if (fabs(F[i + a * k]) > best) { best = fabs(F[i + a * k]); p = i; }
      flag[1] = p;
      flag[0] = F[p + a * k] == 0.0 ? 1 : 0;
    }
    __syncthreads();
    if (flag[0]) return false;
    const int p = flag[1];
    if (p != k) {
      for (int j = threadIdx.x; j < a; j += blockDim.x) { const double t = F[k + a * j]; F[k + a * j] = F[p + a * j]; F[p + a * j] = t; }
      for (int j = threadIdx.x; j < nn; j += blockDim.x) { const double t = X[k + a * j]; X[k + a * j] = X[p + a * j]; X[p + a * j] = t; }
    }
    __syncthreads();
    const double dk = F[k + a * k];
    for (int i = k + 1 + threadIdx.x; i < a; i += blockDim.x) F[i + a * k] /= dk;
    __syncthreads();
    const int r = a - k - 1;
    for (int e = threadIdx.x; e < r * r; e += blockDim.x) {
      const int i = k + 1 + e % r, j = k + 1 + e / r;
      F[i + a * j] -= F[i + a * k] * F[k + a * j];
    }
    __syncthreads();
  }
  return true;
}

// W[alpha, alpha] Z = W[alpha, nu] for every step with a separator, one CTA per step
__global__ void __launch_bounds__(kSolveThreads) solve_kernel(int64_t N, const double* W, StepTable st, double* Zg,
                                                              int* fallbacks) {
  extern __shared__ double sm[];
  __shared__ int flag[2];
  __shared__ int nonfinite;
  const int64_t t = blockIdx.x;
  const int64_t* s = st.steps + 6 * t;
  const int64_t lo = s[0];
  const int nn = (int)(s[1] - s[0]), a = (int)(s[3] - s[2]);
  if (lo == 0 || nn == 0 || a == 0) return;
  const int64_t* al = st.idx + s[2];
  double* F = sm;                  // a x a
  double* V = F + a * a;           // a x a: eigenvectors
  double* X = V + a * a;           // a x nn: right-hand side, then Z
  double* B = X + a * nn;          // a x nn: right-hand side kept for the fallbacks
  double* lam = B + a * nn;        // a
  auto load_F = [&]() {
    for (int e = threadIdx.x; e < a * a; e += blockDim.x) F[e] = W[al[e % a] + N * al[e / a]];
  };
  load_F();
  for (int e = threadIdx.x; e < a * nn; e += blockDim.x) {
    const double b = W[al[e % a] + N * (lo + e / a)];
    B[e] = b;
    X[e] = b;
  }
  if (threadIdx.x == 0) nonfinite = 0;
  __syncthreads();
  bool ok = block_cholesky(F, a, flag);
  if (ok) {
    for (int j = threadIdx.x; j < nn; j += blockDim.x) {   // L L' z = b, one column per thread
      double* x = X + a * j;
      for (int i = 0; i < a; ++i) {
        double v = x[i];
        for (int k = 0; k < i; ++k) v -= F[i + a * k] * x[k];
        x[i] = v / F[i + a * i];
      }
      for (int i = a - 1; i >= 0; --i) {
        double v = x[i];
        for (int k = i + 1; k < a; ++k) v -= F[k + a * i] * x[k];
        x[i] = v / F[i + a * i];
      }
    }
  } else {
    __syncthreads();
    load_F();
    __syncthreads();
    ok = block_lu(F, X, a, nn, flag);
    if (ok) {
      for (int j = threadIdx.x; j < nn; j += blockDim.x) {
        double* x = X + a * j;
        for (int i = 0; i < a; ++i) {
          double v = x[i];
          for (int k = 0; k < i; ++k) v -= F[i + a * k] * x[k];
          x[i] = v;
        }
        for (int i = a - 1; i >= 0; --i) {
          double v = x[i];
          for (int k = i + 1; k < a; ++k) v -= F[i + a * k] * x[k];
          x[i] = v / F[i + a * i];
        }
      }
    }
  }
  __syncthreads();
  if (ok) {
    for (int e = threadIdx.x; e < a * nn; e += blockDim.x)
      if (!isfinite(X[e])) nonfinite = 1;
    __syncthreads();
    ok = !nonfinite;
  }
  if (!ok) {
    // pinv(W[alpha, alpha]) W[alpha, nu] through the cyclic Jacobi eigendecomposition W = V diag(lam) V'
    __syncthreads();
    load_F();
    for (int e = threadIdx.x; e < a * a; e += blockDim.x) V[e] = (e % a == e / a) ? 1.0 : 0.0;
    __syncthreads();
    __shared__ double cs[2];
    __shared__ int done;
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
      if (threadIdx.x == 0) {
        double off = 0.0, tot = 0.0;
        for (int q = 0; q < a; ++q)
          for (int p = 0; p < a; ++p) {
            const double f = F[p + a * q] * F[p + a * q];
            tot += f;
            if (p != q) off += f;
          }
        done = !(off > 1e-30 * tot);
      }
      __syncthreads();
      if (done) break;
      for (int p = 0; p < a - 1; ++p)
        for (int q = p + 1; q < a; ++q) {
          if (threadIdx.x == 0) {
            const double apq = F[p + a * q];
            if (apq == 0.0) {
              cs[0] = 1.0; cs[1] = 0.0;
            } else {
              const double th = (F[q + a * q] - F[p + a * p]) / (2.0 * apq);
              const double tn = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
              cs[0] = 1.0 / sqrt(tn * tn + 1.0);
              cs[1] = tn * cs[0];
            }
          }
          __syncthreads();
          const double c = cs[0], sn = cs[1];
          if (sn != 0.0) {
            for (int k = threadIdx.x; k < a; k += blockDim.x) {   // columns: F J, V J
              const double fp = F[k + a * p], fq = F[k + a * q];
              F[k + a * p] = c * fp - sn * fq;
              F[k + a * q] = sn * fp + c * fq;
              const double vp = V[k + a * p], vq = V[k + a * q];
              V[k + a * p] = c * vp - sn * vq;
              V[k + a * q] = sn * vp + c * vq;
            }
            __syncthreads();
            for (int k = threadIdx.x; k < a; k += blockDim.x) {   // rows: J' (F J)
              const double fp = F[p + a * k], fq = F[q + a * k];
              F[p + a * k] = c * fp - sn * fq;
              F[q + a * k] = sn * fp + c * fq;
            }
          }
          __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
      double lmax = 0.0;
      for (int i = 0; i < a; ++i) lmax = fmax(lmax, fabs(F[i + a * i]));
      for (int i = 0; i < a; ++i) lam[i] = fabs(F[i + a * i]) > kPinvRcond * lmax ? 1.0 / F[i + a * i] : 0.0;
      atomicAdd(fallbacks, 1);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < a * nn; e += blockDim.x) {     // X = diag(1/lam) V' B
      const int i = e % a, j = e / a;
      double v = 0.0;
      for (int k = 0; k < a; ++k) v += V[k + a * i] * B[k + a * j];
      X[e] = lam[i] * v;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < a * nn; e += blockDim.x) {     // Z = V X
      const int i = e % a, j = e / a;
      double v = 0.0;
      for (int k = 0; k < a; ++k) v += V[i + a * k] * X[k + a * j];
      Zg[st.z_off[t] + e] = v;
    }
    return;
  }
  for (int e = threadIdx.x; e < a * nn; e += blockDim.x) Zg[st.z_off[t] + e] = X[e];
}

// the cliques in traversal order, a grid barrier after each: W[r, nu] = W[nu, r] = W[r, alpha] Z for r < lo outside
// the clique (a step without a separator starts a new connected component: its block is zero)
__global__ void __launch_bounds__(kThreads) update_kernel(int64_t N, double* W, StepTable st, const double* Zg) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  extern __shared__ double sm[];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = 0; t < st.n_steps; ++t) {
    const int64_t* s = st.steps + 6 * t;
    const int64_t lo = s[0];
    const int nn = (int)(s[1] - s[0]), a = (int)(s[3] - s[2]), nk = (int)(s[5] - s[2]);
    if (lo == 0 || nn == 0) continue;
    double* Z = sm;
    int64_t* known = reinterpret_cast<int64_t*>(Z + a * nn);   // alpha, then the other clique members below lo
    for (int e = threadIdx.x; e < a * nn; e += blockDim.x) Z[e] = Zg[st.z_off[t] + e];
    for (int e = threadIdx.x; e < nk; e += blockDim.x) known[e] = st.idx[s[2] + e];
    __syncthreads();
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < lo; r += stride) {
      bool inside = false;
      for (int e = 0; e < nk; ++e) inside |= known[e] == r;
      if (inside) continue;
      for (int j = 0; j < nn; ++j) {
        double v = 0.0;
        for (int p = 0; p < a; ++p) v += W[r + N * known[p]] * Z[p + a * j];
        W[r + N * (lo + j)] = v;
        W[lo + j + N * r] = v;
      }
    }
    grid.sync();
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------
static inline void fail(int code, const std::string& msg) { throw EngineError{code, msg}; }

// a validated completion schedule on the device
struct Cone {
  int64_t N = 0, row_offset = 0, n_steps = 0, z_total = 0, max_lo = 0;
  int square = 0;                 // the rows are the N^2 entries of a PsdCone (traditional transformation only)
  size_t smem_solve = 0, smem_update = 0;
  DevBuf<int64_t> new_of, steps, idx, z_off;
  StepTable table() const { return StepTable{n_steps, steps.p, idx.p, z_off.p}; }
};

// checks of one schedule (chordal.validate_schedule); m_orig < 0: a bare matrix.  square_ok: the traditional
// transformation, whose cones may have the square PsdCone layout (dim = N^2).
static void check_schedule(const cosmo_b200_completion& c, int64_t m_orig, int64_t k, bool square_ok = false) {
  const std::string where = m_orig >= 0 ? "decomposition: cone " + std::to_string(k) + ": " : "psd_complete: ";
  const int64_t N = c.N;
  if (N < 1 || N >= (1LL << 31) || !c.new_of || c.n_steps < 0 || c.n_idx < 0 || (c.n_steps && !c.steps) ||
      (c.n_idx && !c.idx))
    fail(COSMO_B200_ERR_INVALID, where + "N, the step count or an array pointer is invalid");
  if (m_orig >= 0) {
    const bool square = c.dim == N * N && N > 1;
    if (square && !square_ok)
      fail(COSMO_B200_ERR_UNSUPPORTED, where + "the square PsdCone layout is not supported by the compact transformation");
    if ((!square && c.dim != N * (N + 1) / 2) || c.row_offset < 0 || c.row_offset + c.dim > m_orig)
      fail(COSMO_B200_ERR_INVALID, where + "the rows of the cone are out of range");
  }
  std::vector<char> hit(N, 0);
  for (int64_t i = 0; i < N; ++i) {
    const int64_t v = c.new_of[i];
    if (v < 0 || v >= N || hit[v]) fail(COSMO_B200_ERR_INVALID, where + "new_of is not a permutation of 0..N-1");
    hit[v] = 1;
  }
  int64_t lo_expect = 0;
  for (int64_t t = 0; t < c.n_steps; ++t) {
    const int64_t* s = c.steps + 6 * t;
    if (s[0] != lo_expect || s[1] < s[0] || s[1] > N)
      fail(COSMO_B200_ERR_INVALID, where + "step " + std::to_string(t) + " does not continue the leading block");
    if (!(0 <= s[2] && s[2] <= s[3] && s[3] == s[4] && s[4] <= s[5] && s[5] <= c.n_idx))
      fail(COSMO_B200_ERR_INVALID, where + "step " + std::to_string(t) + " has inconsistent index ranges");
    for (int64_t e = s[2]; e < s[5]; ++e)
      if (c.idx[e] < 0 || c.idx[e] >= s[0])
        fail(COSMO_B200_ERR_INVALID, where + "step " + std::to_string(t) + " refers to a vertex outside the leading block");
    lo_expect = s[1];
  }
}

static void upload_cone(Cone& dst, const cosmo_b200_completion& c, cudaStream_t st) {
  dst.N = c.N;
  dst.row_offset = c.row_offset;
  dst.square = c.dim == c.N * c.N && c.N > 1;
  dst.n_steps = c.n_steps;
  std::vector<int64_t> zoff(std::max<int64_t>(c.n_steps, 1), 0);
  int64_t z = 0, amax = 0, nnmax = 0, nkmax = 0;
  dst.max_lo = 0;
  for (int64_t t = 0; t < c.n_steps; ++t) {
    const int64_t* s = c.steps + 6 * t;
    const int64_t nn = s[1] - s[0], a = s[3] - s[2];
    zoff[t] = z;
    if (s[0] > 0 && nn > 0) {
      z += a * nn;
      amax = std::max(amax, a);
      nnmax = std::max(nnmax, nn);
      nkmax = std::max(nkmax, s[5] - s[2]);
      dst.smem_solve = std::max(dst.smem_solve, sizeof(double) * (size_t)(2 * a * a + 2 * a * nn + a));
      dst.smem_update = std::max(dst.smem_update, sizeof(double) * (size_t)(a * nn) + sizeof(int64_t) * (size_t)(s[5] - s[2]));
      dst.max_lo = std::max(dst.max_lo, s[0]);
    }
  }
  if (dst.smem_solve > kMaxSmem || dst.smem_update > kMaxSmem)
    fail(COSMO_B200_ERR_UNSUPPORTED, "completion: a separator of " + std::to_string(amax) + " vertices with a residual of " +
                                         std::to_string(nnmax) + " does not fit in shared memory");
  dst.z_total = z;
  dst.new_of.alloc(c.N, false);
  dst.new_of.upload(c.new_of, c.N, st);
  dst.steps.alloc(std::max<int64_t>(6 * c.n_steps, 1), false);
  dst.steps.upload(c.steps, 6 * c.n_steps, st);
  dst.idx.alloc(std::max<int64_t>(c.n_idx, 1), false);
  dst.idx.upload(c.idx, c.n_idx, st);
  dst.z_off.alloc(zoff.size(), false);
  dst.z_off.upload(zoff.data(), zoff.size(), st);
  CUDA_TRY(cudaStreamSynchronize(st));
}

static inline int grid_for(int64_t work) {
  return (int)std::min<int64_t>(std::max<int64_t>((work + kThreads - 1) / kThreads, 1), 8192);
}

// The completion of one cone on W (already in the traversal numbering).  z: at least cone.z_total doubles.
static void complete(const Cone& cone, double* W, double* z, int* fallbacks, cudaStream_t st, int device) {
  if (cone.max_lo == 0) return;
  if (cone.smem_solve > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cone.smem_solve));
  if (cone.smem_update > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cone.smem_update));
  solve_kernel<<<(unsigned)cone.n_steps, kSolveThreads, cone.smem_solve, st>>>(cone.N, W, cone.table(), z, fallbacks);
  CUDA_TRY(cudaGetLastError());
  int sms = 0, per_sm = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, update_kernel, kThreads, cone.smem_update));
  if (per_sm < 1) fail(COSMO_B200_ERR_CUDA, "completion: the update kernel does not fit on an SM");
  // a grid barrier costs more the more CTAs take part: at most two per SM, and no more than the rows need
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)std::min(per_sm, 2) * sms,
                                                               (cone.max_lo + kThreads - 1) / kThreads));
  int64_t N = cone.N;
  StepTable tab = cone.table();
  const double* zc = z;
  void* args[] = {&N, &W, &tab, &zc};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)update_kernel, dim3(grid), dim3(kThreads), args, cone.smem_update, st));
}

// Allocate `buf` for `count` doubles unless it holds that many already; ERR_ALLOC names the matrix side.
static void ensure(DevBuf<double>& buf, size_t count, int64_t N) {
  if (buf.p && buf.n >= count) return;
  try {
    buf.alloc(count, false);
  } catch (const EngineError& e) {
    if (e.code != COSMO_B200_ERR_ALLOC) throw;
    fail(COSMO_B200_ERR_ALLOC, "completion: the dense workspace of N = " + std::to_string(N) + " (" +
                                   std::to_string(8.0 * (double)count / 1e9) + " GB) does not fit in device memory");
  }
}

// The decomposition map of one engine and the buffers of its reverse.
class Reverse {
 public:
  bool has_map() const { return set_; }

  void clear() {
    set_ = false;
    traditional_ = false;
    cones_.clear();
  }

  // traditional: the map of the traditional transformation (cosmo_b200_set_decomposition_noncompact): mu_src must be
  // NULL, mu is the mean of the listed rows, and a cone may have the square PsdCone layout
  void set(const cosmo_b200_decomposition& d, int64_t n, int64_t m, cudaStream_t st, bool traditional = false) {
    clear();
    if (d.n != n || d.m != m)
      fail(COSMO_B200_ERR_INVALID, "decomposition: n, m (" + std::to_string(d.n) + ", " + std::to_string(d.m) +
                                       ") are not the engine's (" + std::to_string(n) + ", " + std::to_string(m) + ")");
    if (d.n_orig < 0 || d.n_orig > n || d.m_orig < 0 || d.n_plain < 0 || d.n_rows < 0 || d.n_cones < 0 ||
        (d.n_plain && !d.plain) || (d.n_rows && (!d.row || !d.s_ptr || (!traditional && !d.mu_src))) ||
        (d.n_cones && !d.cones))
      fail(COSMO_B200_ERR_INVALID, "decomposition: bad dimensions or a missing array");
    if (traditional && d.mu_src)
      fail(COSMO_B200_ERR_INVALID, "decomposition: mu_src must be NULL for the traditional transformation (mu is the mean)");
    // plain blocks and decomposed rows: in range, and no original row written twice
    std::vector<std::pair<int64_t, int64_t>> spans;
    std::vector<int64_t> pref(d.n_plain + 1, 0);
    for (int64_t b = 0; b < d.n_plain; ++b) {
      const int64_t old = d.plain[3 * b], nw = d.plain[3 * b + 1], dim = d.plain[3 * b + 2];
      if (old < 0 || nw < 0 || dim < 0 || old + dim > d.m_orig || nw + dim > m)
        fail(COSMO_B200_ERR_INVALID, "decomposition: plain block " + std::to_string(b) + " is out of range");
      if (dim) spans.push_back({old, old + dim});
      pref[b + 1] = pref[b] + dim;
    }
    std::sort(spans.begin(), spans.end());
    for (size_t i = 1; i < spans.size(); ++i)
      if (spans[i].first < spans[i - 1].second) fail(COSMO_B200_ERR_INVALID, "decomposition: plain blocks overlap");
    const int64_t nnz = d.n_rows ? d.s_ptr[d.n_rows] : 0;
    if (d.n_rows && (d.s_ptr[0] != 0 || nnz < 0 || (nnz && !d.s_src)))
      fail(COSMO_B200_ERR_INVALID, "decomposition: s_ptr is inconsistent");
    for (int64_t i = 0; i < d.n_rows; ++i) {
      const int64_t r = d.row[i];
      if (r < 0 || r >= d.m_orig || (i && r <= d.row[i - 1]))
        fail(COSMO_B200_ERR_INVALID, "decomposition: rows out of range or not increasing");
      auto it = std::upper_bound(spans.begin(), spans.end(), std::make_pair(r, INT64_MAX));
      if (it != spans.begin() && r < std::prev(it)->second)
        fail(COSMO_B200_ERR_INVALID, "decomposition: row " + std::to_string(r) + " lies in a plain block");
      if (d.s_ptr[i + 1] <= d.s_ptr[i] || d.s_ptr[i + 1] > nnz) fail(COSMO_B200_ERR_INVALID, "decomposition: s_ptr is inconsistent");
      for (int64_t p = d.s_ptr[i]; p < d.s_ptr[i + 1]; ++p)
        if (d.s_src[p] < 0 || d.s_src[p] >= m) fail(COSMO_B200_ERR_INVALID, "decomposition: s_src out of range");
      if (!traditional && d.mu_src[i] != d.s_src[d.s_ptr[i + 1] - 1])
        fail(COSMO_B200_ERR_INVALID, "decomposition: mu_src of row " + std::to_string(r) + " is not its last clique row");
    }
    for (int64_t k = 0; k < d.n_cones; ++k) check_schedule(d.cones[k], d.m_orig, k, traditional);

    n_orig_ = d.n_orig; m_orig_ = d.m_orig; n_rows_ = d.n_rows; n_plain_ = d.n_plain; plain_rows_ = pref[d.n_plain];
    auto up = [&](DevBuf<int64_t>& dst, const int64_t* src, int64_t count) {
      dst.alloc(std::max<int64_t>(count, 1), false);
      dst.upload(src, count, st);
    };
    up(plain_, d.plain, 3 * d.n_plain);
    up(plain_pref_, pref.data(), d.n_plain + 1);
    up(row_, d.row, d.n_rows);
    up(s_ptr_, d.s_ptr, d.n_rows ? d.n_rows + 1 : 0);
    up(s_src_, d.s_src, nnz);
    up(mu_src_, d.mu_src, traditional ? 0 : d.n_rows);
    cones_ = std::vector<Cone>(d.n_cones);
    for (int64_t k = 0; k < d.n_cones; ++k) upload_cone(cones_[k], d.cones[k], st);
    CUDA_TRY(cudaStreamSynchronize(st));
    traditional_ = traditional;
    set_ = true;
  }

  template <typename T>
  void run(const T* x, const T* s, const T* mu, const T* D, const T* E, double c, bool complete_dual, void* hx, void* hs,
           void* hmu, int64_t* stats, cudaStream_t st, int device, bool negate_mu = false) {
    if (!set_) fail(COSMO_B200_ERR_INVALID, "reverse_decomposition: no decomposition map (cosmo_b200_set_decomposition)");
    ensure(x_, std::max<int64_t>(n_orig_, 1), 0);
    ensure(s_, std::max<int64_t>(m_orig_, 1), 0);
    ensure(mu_, std::max<int64_t>(m_orig_, 1), 0);
    const bool completing = complete_dual && hmu && !cones_.empty();
    int64_t nmax = 0, zmax = 1;
    for (const Cone& k : cones_) { nmax = std::max(nmax, k.N); zmax = std::max(zmax, k.z_total); }
    if (completing) {
      ensure(W_, (size_t)nmax * nmax, nmax);
      ensure(z_, zmax, nmax);
    }
    if (!cnt_.p) cnt_.alloc(1);
    ev_[0].create();
    ev_[1].create();
    CUDA_TRY(cudaMemsetAsync(cnt_.p, 0, sizeof(int), st));
    CUDA_TRY(cudaEventRecord(ev_[0], st));
    if (hs) CUDA_TRY(cudaMemsetAsync(s_.p, 0, m_orig_ * sizeof(double), st));
    if (hmu) CUDA_TRY(cudaMemsetAsync(mu_.p, 0, m_orig_ * sizeof(double), st));
    GatherArgs<T> a{n_orig_, n_rows_, n_plain_, plain_rows_, x, s, mu, D, E, c, row_.p, s_ptr_.p, s_src_.p, mu_src_.p,
                    plain_.p, plain_pref_.p, traditional_ ? 1 : 0, hx ? x_.p : nullptr, hs ? s_.p : nullptr,
                    hmu ? mu_.p : nullptr};
    gather_kernel<T><<<grid_for(n_orig_ + n_rows_ + plain_rows_), kThreads, 0, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    if (completing) {
      for (const Cone& k : cones_) {
        double* v = mu_.p + k.row_offset;
        scatter_kernel<<<grid_for(k.N * (k.N + 1) / 2), kThreads, 0, st>>>(k.N, v, k.new_of.p, W_.p, k.square);
        CUDA_TRY(cudaGetLastError());
        complete(k, W_.p, z_.p, cnt_.p, st, device);
        gather_back_kernel<<<grid_for(k.square ? k.N * k.N : k.N * (k.N + 1) / 2), kThreads, 0, st>>>(k.N, k.new_of.p, W_.p,
                                                                                                       v, k.square);
        CUDA_TRY(cudaGetLastError());
      }
    }
    if (hmu && negate_mu) {
      negate_kernel<<<grid_for(m_orig_), kThreads, 0, st>>>(m_orig_, mu_.p);
      CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaEventRecord(ev_[1], st));
    if (hx) CUDA_TRY(cudaMemcpyAsync(hx, x_.p, n_orig_ * sizeof(double), cudaMemcpyDefault, st));
    if (hs) CUDA_TRY(cudaMemcpyAsync(hs, s_.p, m_orig_ * sizeof(double), cudaMemcpyDefault, st));
    if (hmu) CUDA_TRY(cudaMemcpyAsync(hmu, mu_.p, m_orig_ * sizeof(double), cudaMemcpyDefault, st));
    int fallbacks = 0;
    CUDA_TRY(cudaMemcpyAsync(&fallbacks, cnt_.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
    if (stats) {
      stats[0] = completing ? (int64_t)cones_.size() : 0;
      stats[1] = fallbacks;
      stats[2] = W_.p ? (int64_t)(W_.n * sizeof(double)) : 0;
      stats[3] = (int64_t)llround(1000.0 * ms);   // microseconds
    }
    last_ms_ = ms;
  }

  double last_ms() const { return last_ms_; }

 private:
  bool set_ = false, traditional_ = false;
  int64_t n_orig_ = 0, m_orig_ = 0, n_rows_ = 0, n_plain_ = 0, plain_rows_ = 0;
  DevBuf<int64_t> plain_, plain_pref_, row_, s_ptr_, s_src_, mu_src_;
  std::vector<Cone> cones_;
  DevBuf<double> x_, s_, mu_, W_, z_;
  DevBuf<int> cnt_;
  Event ev_[2];
  double last_ms_ = 0.0;
};

}  // namespace rev
}  // namespace cosmo
