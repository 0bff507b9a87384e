// aa.cuh -- safeguarded Anderson acceleration of the ADMM operator (SURVEY.md 8f-1):
// AndersonAccelerator{T, Type2{QRDecomp}, RestartedMemory, NoRegularizer}, the reference's default
// accelerator (settings.jl:136-138), driven through acceleration_pre!/post! (accelerator_interface.jl:58-114).
//
// The arithmetic lives in COSMOAccelerators.jl (not part of the reference tree); it is restated here from the
// published method -- type-II Anderson acceleration, least squares min |f - F eta| by a QR factorisation of
// F = [f_k - f_{k-1}] that is extended one column per iteration (modified Gram-Schmidt), memory emptied when
// its `mem` columns are full.  Iterate-level parity with the package is therefore UNPINNED; the CPU oracle
// holds the same restatement and the reference's behavioural tests (AccelerationTests) are reproduced.
//
// All vectors have the length of the operator variable w = [w_x; w_s].  On a row-sharded run w_x is replicated:
// inner products run over [lo, dim) with lo = 0 on rank 0 and lo = n elsewhere, followed by an allreduce, so
// every rank holds the same R and eta and applies the same update to its copy of w_x.
#pragma once
#include <cmath>

#include "common.cuh"

namespace cosmo {

// AA_F2 and AA_FACC2 hold the AA_SSQ scaled sums of squares of aa_ssq_add each
enum { AA_SSQ = 3, AA_F2 = 0, AA_FACC2 = AA_SSQ, AA_FLAG = 2 * AA_SSQ, AA_NRM2 = AA_FLAG + 1, AA_SC_COUNT = 8 };

// The safeguard's two norms |f|_2 and |f_acc|_2 (accelerator_interface.jl:90,120-123) are the reference's norm(f, 2),
// which rescales and neither overflows nor underflows.  A plain sum of squares in T overflows once |f|_2 passes
// sqrt(max(T)) (1.8e19 in float32), and the test nrm_f_acc > tol * nrm_f then never declines.  So each entry goes to
// one of three sums of squares by its magnitude, with the thresholds and power-of-two scales of LAPACK's dnrm2 (Blue's
// algorithm, la_constants.f90): x^2 for tsml <= |x| <= tbig, (x sbig)^2 above, (x ssml)^2 below.  Scaling by a power of
// two is exact, no sum overflows or underflows to zero for any finite entry of T, and the three are plain sums, so a
// sharded allreduce adds them like any other.  aa_norm combines them on the host.  A NaN entry lands in the middle sum.
template <typename T> struct AaBlue;
template <> struct AaBlue<double> {
  static constexpr double tsml = 0x1p-511, tbig = 0x1p486, ssml = 0x1p537, sbig = 0x1p-538;
};
template <> struct AaBlue<float> {
  static constexpr float tsml = 0x1p-63f, tbig = 0x1p52f, ssml = 0x1p75f, sbig = 0x1p-76f;
};

template <typename T>
__device__ __forceinline__ void aa_ssq_add(T (&acc)[AA_SSQ], T x) {
  const T a = tabs(x);
  if (a > AaBlue<T>::tbig) {
    const T y = x * AaBlue<T>::sbig;
    acc[1] += y * y;
  } else if (a < AaBlue<T>::tsml) {
    const T y = x * AaBlue<T>::ssml;
    acc[2] += y * y;
  } else {
    acc[0] += x * x;
  }
}

// |x|_2 from the AA_SSQ sums of aa_ssq_add, in double.  Only the middle sum is set for every vector whose entries lie in
// [tsml, tbig] or are zero, and the result is then sqrt of that sum, as a single sum of squares gives.  NaN when a sum is.
template <typename T>
inline double aa_norm(const T* s) {
  const double mid = sqrt((double)s[0]), big = sqrt((double)s[1]) / (double)AaBlue<T>::sbig,
               sml = sqrt((double)s[2]) / (double)AaBlue<T>::ssml;
  if (mid != mid || big != big || sml != sml) return NAN;
  return std::hypot(std::hypot(mid, big), sml);
}

// CA.update! of every variant: f = x - g; after a restart only (g_last, f_last and, for Type1, x_last) are stored;
// otherwise G[:, j] = g - g_last, F[:, j] = f - f_last and, for Type1 (Xj != nullptr), X[:, j] = x - x_last.
// F lives in Q; the QR variant orthogonalises the new column afterwards.
// out[0:AA_SSQ] = the scaled sums of squares of f over [lo, dim) (the safeguard's reference norm, accelerator_interface.jl:90).
template <typename T>
__global__ void __launch_bounds__(kBlock) aa_hist_kernel(int dim, int lo, const T* __restrict__ g, const T* __restrict__ x,
                                                         T* __restrict__ f, T* __restrict__ f_last, T* __restrict__ g_last,
                                                         T* __restrict__ x_last, T* __restrict__ Gj, T* __restrict__ Fj,
                                                         T* __restrict__ Xj, int init, RedBuf<T> rb) {
  T accS[AA_SSQ] = {0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) {
    const T gi = g[i], xi = x[i];
    const T fi = xi - gi;
    f[i] = fi;
    if (!init) {
      Gj[i] = gi - g_last[i];
      Fj[i] = fi - f_last[i];
      if (Xj) Xj[i] = xi - x_last[i];
    }
    g_last[i] = gi;
    f_last[i] = fi;
    if (x_last) x_last[i] = xi;
    if (i >= lo) aa_ssq_add(accS, fi);
  }
  reduce_and_finalize<T, AA_SSQ, 0>(accS, (const T*)nullptr, rb, NoFin());
}

// One modified Gram-Schmidt step on the new column q:
//   q -= r_prev * Qp   (skipped when Qp == nullptr),   out[0] = <Qi, q>  (or |q|^2 when Qi == nullptr)
template <typename T>
__global__ void __launch_bounds__(kBlock) aa_mgs_kernel(int dim, int lo, T* __restrict__ q, const T* __restrict__ Qp,
                                                        const T* __restrict__ r_prev, const T* __restrict__ Qi, RedBuf<T> rb) {
  T accS[1] = {0};
  const T r = Qp ? *r_prev : T(0);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) {
    T qi = q[i];
    if (Qp) { qi -= r * Qp[i]; q[i] = qi; }
    if (i >= lo) accS[0] += (Qi ? Qi[i] : qi) * qi;
  }
  reduce_and_finalize<T, 1, 0>(accS, (const T*)nullptr, rb, NoFin());
}

// R[j,j] = sqrt(|q|^2) ; q /= R[j,j]
template <typename T>
__global__ void __launch_bounds__(kBlock) aa_normalize_kernel(int dim, T* __restrict__ q, const T* __restrict__ nrm2, T* __restrict__ rjj) {
  const T r = sqrt(*nrm2);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) q[i] = q[i] / r;
  if (blockIdx.x == 0 && threadIdx.x == 0) *rjj = r;
}

// out[c] = <Q[:, c0 + c], f>, c < ncols <= 8
template <typename T>
__global__ void __launch_bounds__(kBlock) aa_qtf_kernel(int dim, int lo, const T* __restrict__ f, const T* __restrict__ Q, size_t ld,
                                                        int c0, int ncols, RedBuf<T> rb) {
  T accS[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) {
    const T fi = f[i];
#pragma unroll
    for (int c = 0; c < 8; ++c)
      if (c < ncols) accS[c] += Q[(size_t)(c0 + c) * ld + i] * fi;
  }
  reduce_and_finalize<T, 8, 0>(accS, (const T*)nullptr, rb, NoFin());
}

// Back substitution R[0:l,0:l] eta = Q'f (in place; R column-major with leading dimension mem) and the
// acceptance test of the candidate: finite, non-singular, |eta|_2 <= 1e4.  flag[0] = 1 accepted / 0 rejected.
template <typename T>
__global__ void aa_solve_kernel(const T* __restrict__ R, int mem, int l, T* __restrict__ eta, T* __restrict__ flag) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  bool ok = true;
  for (int i = l - 1; i >= 0; --i) {
    T v = eta[i];
    for (int k = i + 1; k < l; ++k) v -= R[(size_t)k * mem + i] * eta[k];
    const T d = R[(size_t)i * mem + i];
    if (d == T(0) || !isfinite(d)) ok = false;
    eta[i] = v / d;
  }
  T nrm2 = 0;
  for (int i = 0; i < l; ++i) nrm2 += eta[i] * eta[i];
  const T nrm = sqrt(nrm2);
  if (!isfinite(nrm) || nrm > T(1e4)) ok = false;
  flag[0] = ok ? T(1) : T(0);
}

// CA.accelerate!: w -= G[:, 0:l] eta, only if the candidate was accepted
template <typename T>
__global__ void __launch_bounds__(kBlock) aa_apply_kernel(int dim, T* __restrict__ w, const T* __restrict__ G, size_t ld, int l,
                                                          const T* __restrict__ eta, const T* __restrict__ flag) {
  if (*flag == T(0)) return;
  __shared__ T e[32];
  if (threadIdx.x < l) e[threadIdx.x] = eta[threadIdx.x];
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) {
    T v = w[i];
    for (int c = 0; c < l; ++c) v -= G[(size_t)c * ld + i] * e[c];
    w[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The other variants of anderson_accelerator.jl: AndersonAccelerator{T, Type2{NormalEquations} | Type1,
// RollingMemory | RestartedMemory, NoRegularizer | TikonovRegularizer | FrobeniusNormRegularizer}.
// Restated from the published methods (type-II: Walker & Ni 2011; type-I and its Frobenius-norm regularisation:
// Fu, Zhang & Boyd 2020), parity with COSMOAccelerators.jl UNPINNED like the QR variant above.  With the history
// columns X_j = x - x_last, F_j = f - f_last, G_j = g - g_last each iteration solves the l x l system
//   Type2{NormalEquations}: M = F'F, rhs = F'f        Type1: M = X'F, rhs = X'f
// (M + shift I) eta = rhs by LU with partial pivoting, shift = lambda (Tikonov) or lambda (|A|_F^2 + |B|_F^2) for
// M = A'B (Frobenius), and the candidate is g - G eta.  M is kept on the device in physical column order; a new
// column j refreshes row j and column j of M against the whole window (RollingMemory overwrites column iter mod mem).
// ---------------------------------------------------------------------------------------------------------------
enum { AA_GRAM_COLS = 8, AA_GRAM_NR = 3 * AA_GRAM_COLS + 2, AA_GRAM_MAX_CHUNKS = 4 };

// The fused Gram + right-hand-side pass over window columns c = c0 .. c0 + ncols - 1 (ncols <= 8) of A (X for
// Type1, F for Type2) and B = F, the new column j and f; each history column is read once:
//   out[c] = <A_j, B_c> (row j of M),  out[8 + c] = <A_c, B_j> (column j of M, Type1 only),  out[16 + c] = <A_c, f>,
//   out[24] = |A_j|^2,  out[25] = |B_j|^2 (Type1 only; the Frobenius regulariser).   Sums over [lo, dim).
template <typename T, bool TYPE1>
__global__ void __launch_bounds__(kBlock) aa_gram_kernel(int dim, int lo, const T* __restrict__ A, const T* __restrict__ B,
                                                         size_t ld, int j, int c0, int ncols, const T* __restrict__ f,
                                                         RedBuf<T> rb) {
  T acc[AA_GRAM_NR];
#pragma unroll
  for (int k = 0; k < AA_GRAM_NR; ++k) acc[k] = T(0);
  const T* Aj = A + (size_t)j * ld;
  const T* Bj = B + (size_t)j * ld;
  for (int i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) {
    const T aj = Aj[i], fi = f[i];
    const T bj = TYPE1 ? Bj[i] : aj;
#pragma unroll
    for (int c = 0; c < AA_GRAM_COLS; ++c)
      if (c < ncols) {
        const T a = A[(size_t)(c0 + c) * ld + i];
        const T b = TYPE1 ? B[(size_t)(c0 + c) * ld + i] : a;
        acc[c] += aj * b;
        if (TYPE1) acc[AA_GRAM_COLS + c] += a * bj;
        acc[2 * AA_GRAM_COLS + c] += a * fi;
      }
    acc[3 * AA_GRAM_COLS] += aj * aj;
    if (TYPE1) acc[3 * AA_GRAM_COLS + 1] += bj * bj;
  }
  reduce_and_finalize<T, AA_GRAM_NR, 0, NoFin, kWarpsPerBlock, AA_GRAM_NR>(acc, (const T*)nullptr, rb, NoFin());
}

// One warp (lane r owns row r, l <= 32).  Scatters the reduced Gram pass `gsc` (AA_GRAM_NR scalars per chunk of 8
// columns) into row and column j of M (row-major, leading dimension mem) and the column norms; with `solve`, factors
// M[0:l, 0:l] + shift I by LU with partial pivoting (first largest |pivot|), solves for eta and applies the
// acceptance test of aa_solve_kernel: no zero or non-finite pivot, eta finite, |eta|_2 <= 1e4.  flag[0] = 1 / 0.
// reg: 0 none, 1 Tikonov (shift = lambda), 2 Frobenius (shift = lambda sum_c (nrmA[c] + nrmB[c])).
template <typename T>
__global__ void __launch_bounds__(32) aa_ne_solve_kernel(const T* __restrict__ gsc, T* __restrict__ M, T* __restrict__ nrmA,
                                                         T* __restrict__ nrmB, int mem, int j, int l, int type1, int reg,
                                                         T lambda, int solve, T* __restrict__ eta, T* __restrict__ flag) {
  __shared__ T S[32][33];
  __shared__ T rhs[32];
  const int r = threadIdx.x;
  if (r < l) {
    const T* o = gsc + (r / AA_GRAM_COLS) * AA_GRAM_NR;
    const int k = r % AA_GRAM_COLS;
    M[(size_t)j * mem + r] = o[k];
    if (r != j) M[(size_t)r * mem + j] = type1 ? o[AA_GRAM_COLS + k] : o[k];
    rhs[r] = o[2 * AA_GRAM_COLS + k];
  }
  if (r == 0) {
    nrmA[j] = gsc[3 * AA_GRAM_COLS];
    nrmB[j] = type1 ? gsc[3 * AA_GRAM_COLS + 1] : gsc[3 * AA_GRAM_COLS];
  }
  __threadfence_block();
  __syncwarp();
  if (!solve) return;
  T shift = T(0);
  if (reg == 1) shift = lambda;
  if (reg == 2) shift = lambda * warp_sum(r < l ? nrmA[r] + nrmB[r] : T(0));
  bool ok = true;
  if (r < l) {
    for (int c = 0; c < l; ++c) {
      const T v = M[(size_t)r * mem + c] + (c == r ? shift : T(0));
      S[r][c] = v;
      if (!isfinite(v)) ok = false;
    }
    if (!isfinite(rhs[r])) ok = false;
  }
  ok = __all_sync(0xffffffffu, ok);
  __syncwarp();
  for (int k = 0; k < l && ok; ++k) {
    T v = (r >= k && r < l) ? tabs(S[r][k]) : T(-1);
    if (v != v) v = T(INFINITY);
    int idx = r;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const T ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
    }
    const T piv = S[idx][k];
    __syncwarp();   // every lane has read the pivot before the row swap below rewrites S[idx][k]
    if (piv == T(0) || !isfinite(piv)) { ok = false; break; }
    if (idx != k) {
      if (r < l) { const T t = S[k][r]; S[k][r] = S[idx][r]; S[idx][r] = t; }
      if (r == 0) { const T t = rhs[k]; rhs[k] = rhs[idx]; rhs[idx] = t; }
    }
    __syncwarp();
    if (r > k && r < l) {
      const T fct = S[r][k] / S[k][k];
      S[r][k] = fct;
      for (int c = k + 1; c < l; ++c) S[r][c] -= fct * S[k][c];
      rhs[r] -= fct * rhs[k];
    }
    __syncwarp();
  }
  if (r != 0) return;
  if (ok) {
    for (int i = l - 1; i >= 0; --i) {
      T v = rhs[i];
      for (int k = i + 1; k < l; ++k) v -= S[i][k] * rhs[k];
      rhs[i] = v / S[i][i];
    }
    T nrm2 = 0;
    for (int i = 0; i < l; ++i) nrm2 += rhs[i] * rhs[i];
    const T nrm = sqrt(nrm2);
    if (!isfinite(nrm) || nrm > T(1e4)) ok = false;
    for (int i = 0; i < l; ++i) eta[i] = rhs[i];
  }
  flag[0] = ok ? T(1) : T(0);
}

// compute_accelerated_res_norm! (accelerator_interface.jl:120-123): f = w_prev - w, out[0:AA_SSQ] = the scaled sums of
// squares of f (aa_ssq_add)
template <typename T>
__global__ void __launch_bounds__(kBlock) aa_res_kernel(int dim, int lo, const T* __restrict__ w_prev, const T* __restrict__ w,
                                                        T* __restrict__ f, RedBuf<T> rb) {
  T accS[AA_SSQ] = {0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < dim; i += gridDim.x * blockDim.x) {
    const T fi = w_prev[i] - w[i];
    f[i] = fi;
    if (i >= lo) aa_ssq_add(accS, fi);
  }
  reduce_and_finalize<T, AA_SSQ, 0>(accS, (const T*)nullptr, rb, NoFin());
}

}  // namespace cosmo
