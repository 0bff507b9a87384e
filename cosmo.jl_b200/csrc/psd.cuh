// psd.cuh -- PSD-cone projection on the device (kernel K6 of SURVEY.md 2a).
//
// Replaces project!(x, ::PsdCone / ::PsdConeTriangle) (reference
// src/convexset.jl:303-321, 402-412 -> _project! :219-241 -> LAPACK ?syevr
// :163-189 -> rank_k_update! :243-263 -> svec pack/unpack :432-472).
//
// Round-1 eigensolver: cyclic two-sided Jacobi with the round-robin parallel
// ordering, in the cone's own precision (fp64 for Model{Float64}).
//   * small cones (N <= kPsdSmallMax; the clique batch produced by chordal
//     decomposition): ONE CTA PER CONE, matrix and eigenvectors resident in
//     shared memory, every cone of the batch in one launch.
//   * large cones: matrix/eigenvectors in HBM (L2-resident for N <= ~2800),
//     block Jacobi, one (pivot, columns, rows) kernel triple per round.
// The projection keeps eigenpairs with lambda > 0 strictly (convexset.jl:250)
// and rebuilds X+ = sum lambda_k v_k v_k' ; a cone of dim 1 is max(x, 0)
// (convexset.jl:307-308, 404-405).
//
// fp64 note (SURVEY.md H1): this path runs on the FP64 FMA pipe; large cones take
// the int8-sliced tensor-core path of psd_tc.cuh.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "host.cuh"

namespace cosmo {

struct PsdConeDesc {
  int off;       // first row of the cone in s
  int N;         // side of the real symmetric matrix that is diagonalised
  int triangle;  // 1: svec upper triangle (PsdConeTriangle), 0: column-major square (PsdCone),
                 // 2: PsdConeTriangle{T, Complex{T}} (convexset.jl:344-360, 444-490): the Hermitian Nc x Nc matrix
                 //    X = A + iB is handled through its real embedding [[A, -B], [B, A]] of side N = 2 Nc, whose
                 //    projection is the embedding of the projection of X
};

constexpr int kPsdSmallMax = 96;   // 2 * (N+1)^2 * 8 B <= 227 KB shared memory

template <typename T> struct PsdEps;
template <> struct PsdEps<double> { static constexpr double v = 2.220446049250313e-16; };
template <> struct PsdEps<float> { static constexpr double v = 1.1920929e-07; };

// symmetric Schur rotation zeroing a_pq (Golub & Van Loan, Alg. 8.4.1)
template <typename T>
__device__ __forceinline__ void sym_schur(T app, T aqq, T apq, T& c, T& s) {
  const T tau = (aqq - app) / (T(2) * apq);
  const T t = (tau >= T(0)) ? T(1) / (tau + sqrt(T(1) + tau * tau)) : T(1) / (tau - sqrt(T(1) + tau * tau));
  c = T(1) / sqrt(T(1) + t * t);
  s = t * c;
}

// round-robin tournament pairing: round r in [0, Ne-1), slot k in [0, Ne/2)
__device__ __forceinline__ void rr_pair(int Ne, int r, int k, int& p, int& q) {
  const int M = Ne - 1;
  if (k == 0) { p = r; q = M; }
  else { p = (r + k) % M; q = (r - k + M) % M; }
  if (p > q) { int t = p; p = q; q = t; }
}

// position of (i,j), i<=j, in the column-major upper triangle (convexset.jl:432-442)
__device__ __forceinline__ long long svec_pos(int i, int j) { return (long long)j * (j + 1) / 2 + i; }

// Entry (i, j) of the real embedding [[A, -B], [B, A]] (side 2 Nc) of the Hermitian matrix X = A + iB stored as
// PsdConeTriangle{T, Complex{T}} (convexset.jl:444-490): the sqrt 2 scaled real upper triangle column by column,
// followed by the sqrt 2 scaled strictly upper imaginary parts column by column.
template <typename T>
__device__ __forceinline__ T hermitian_embedding_entry(const T* __restrict__ x, int Nc, int i, int j) {
  const T inv_sqrt2 = T(0.70710678118654752440);
  const int I = i % Nc, bi = i / Nc, J = j % Nc, bj = j / Nc;
  const int a = I < J ? I : J, b = I < J ? J : I;
  if (bi == bj) {                                   // A = Re X (symmetric)
    const T v = x[svec_pos(a, b)];
    return (a != b) ? v * inv_sqrt2 : v;
  }
  if (I == J) return T(0);                          // Im X has a zero diagonal
  const T im_ab = x[(long long)Nc * (Nc + 1) / 2 + (long long)b * (b - 1) / 2 + a] * inv_sqrt2;   // Im X[a, b], a < b
  const T b_IJ = (I < J) ? im_ab : -im_ab;          // B = Im X is antisymmetric
  return (bi == 1) ? b_IJ : -b_IJ;                  // lower-left block B, upper-right block -B
}

// s[cone] <- X+ = A+ + i B+ from the projected embedding P (side N = 2 Nc, symmetric; only its upper triangle is read):
// A+ = (P11 + P22) / 2,  B+ = (P21 - P12) / 2
template <typename T, typename TP>
__global__ void __launch_bounds__(kBlock) psd_embedding_store_kernel(PsdConeDesc d, const TP* __restrict__ P, T* __restrict__ s) {
  const int N = d.N, Nc = N >> 1;
  const long long tri = (long long)Nc * (Nc + 1) / 2;
  const double sqrt2 = 1.41421356237309504880;
  const long long total = (long long)Nc * Nc;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const bool imag = e >= tri;
    const long long ee = imag ? e - tri : e;
    long long i, j;
    if (!imag) {          // (i, j), i <= j, of the triangle: ee = j (j + 1) / 2 + i
      j = (long long)((sqrt(8.0 * (double)ee + 1.0) - 1.0) * 0.5);
      while ((j + 1) * (j + 2) / 2 <= ee) ++j;
      while (j * (j + 1) / 2 > ee) --j;
      i = ee - j * (j + 1) / 2;
      const double v = 0.5 * ((double)P[j * N + i] + (double)P[(Nc + j) * N + (Nc + i)]);
      s[d.off + e] = (T)((i == j) ? v : sqrt2 * v);
    } else {              // (i, j), i < j, of the strict triangle: ee = j (j - 1) / 2 + i
      j = (long long)((sqrt(8.0 * (double)ee + 1.0) + 1.0) * 0.5);
      while (j * (j + 1) / 2 <= ee) ++j;
      while (j * (j - 1) / 2 > ee) --j;
      i = ee - j * (j - 1) / 2;
      // P21[i, j] = P[Nc + i, j] = P[j, Nc + i] (upper triangle);  P12[i, j] = P[i, Nc + j]
      const double v = 0.5 * ((double)P[(Nc + i) * N + j] - (double)P[(Nc + j) * N + i]);
      s[d.off + e] = (T)(sqrt2 * v);
    }
  }
}

// ---------------------------------------------------------------------------
// Small cones: one CTA per cone, everything in shared memory.
//   mode 0: s[cone] = Pi_PSD(ws[cone]);  mode 1: lam_max[cone] = max eigenvalue of mat(ws[cone]);
//   mode 2: the eigenpairs of mat(ws[cone]) (symmetrised as in mode 0) into eig (the Jacobian of the projection,
//           solve_adjoint.cuh): Q column-major at eig.Q + eig.q_off[cone], the eigenvalues at eig.lam + eig.lam_off[cone],
//           and the cone counted in eig.kinks when an eigenvalue is within 64 u (1 + max |w_s|) of 0
// mode 0 symmetrizes a square cone as project! does (symmetrize_upper!); mode 1 reads its upper triangle only, as the
// certificate is_pos_def! -> cholesky!(Hermitian(X)) does (convexset.jl:324-336, algebra.jl:226-233): delta y and
// A delta x are not symmetric on the rows of a square cone in general.  In mode 1 a cone whose Jacobi sweeps did not
// converge within max_sweeps gets lam_max = +inf (not certified: the diagonal of a partly rotated matrix can
// underestimate lambda_max) and increments *fail_flag.
// ---------------------------------------------------------------------------
template <typename T>
struct PsdEigOut {
  T* Q = nullptr;
  T* lam = nullptr;
  const long long* q_off = nullptr;
  const int* lam_off = nullptr;
  int* kinks = nullptr;
};

template <typename T>
__global__ void __launch_bounds__(kBlock) psd_small_kernel(const PsdConeDesc* __restrict__ descs, const T* __restrict__ ws,
                                                           T* __restrict__ s, int mode, T* __restrict__ lam_max,
                                                           int max_sweeps, int* __restrict__ fail_flag,
                                                           PsdEigOut<T> eig = PsdEigOut<T>()) {
  extern __shared__ unsigned char smem_raw[];
  const PsdConeDesc d = descs[blockIdx.x];
  const int N = d.N;
  const T* x = ws + d.off;
  if (N == 1) {
    if (threadIdx.x == 0) {
      const T v = x[0];
      if (mode == 0) {
        s[d.off] = (v > T(0)) ? v : ((v != v) ? v : T(0));
      } else if (mode == 1) {
        lam_max[blockIdx.x] = v;
      } else {
        eig.Q[eig.q_off[blockIdx.x]] = T(1);
        eig.lam[eig.lam_off[blockIdx.x]] = v;
        if (tabs(v) <= (T)(64.0 * PsdEps<T>::v) * (T(1) + tabs(v))) atomicAdd(eig.kinks, 1);
      }
    }
    return;
  }
  const int ld = N | 1;  // odd leading dimension: conflict-free row sweeps
  T* A = reinterpret_cast<T*>(smem_raw);
  T* V = A + (size_t)ld * N;
  T* cs = V + (size_t)ld * N;   // 2 * (N/2 + 1): rotation cosines / sines of the round
  __shared__ int pq[kPsdSmallMax + 2];
  __shared__ T red[kWarpsPerBlock];
  __shared__ int rotated;
  __shared__ T thr_sh;
  const T inv_sqrt2 = T(0.70710678118654752440);
  const T sqrt2 = T(1.41421356237309504880);

  // ---- load: X = mat(x) 2^-pe, pe even: the power of two nearest max |X| (exact; every projection is positively
  // homogeneous, so nothing below overflows or underflows whatever the scale of x, and the result is unscaled at the end)
  T mx = 0;
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {
    const int i = e % N, j = e / N;
    T v;
    if (d.triangle == 1) {
      const int a = i < j ? i : j, b = i < j ? j : i;
      v = x[svec_pos(a, b)];
      if (a != b) v *= inv_sqrt2;
    } else if (d.triangle == 2) {
      v = hermitian_embedding_entry(x, N >> 1, i, j);
    } else if (mode == 1) {
      const int a = i < j ? i : j, b = i < j ? j : i;
      v = x[(long long)b * N + a];                                      // Hermitian(X, :U)
    } else {
      v = (x[(long long)j * N + i] + x[(long long)i * N + j]) / T(2);   // symmetrize_upper!, algebra.jl:201-208
    }
    A[i + j * ld] = v;
    V[i + j * ld] = (i == j) ? T(1) : T(0);
    mx = fmax(mx, tabs(v));
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < kWarpsPerBlock; ++w) mx = fmax(mx, red[w]);
  const T mx_in = mx;
  const int pe = pow2_exponent(mx) & ~1;          // even: sqrt(lambda 2^-pe) = sqrt(lambda) 2^(-pe/2) exactly
  const T down = (T)ldexp(1.0, -pe), up = (T)ldexp(1.0, pe);
  __syncthreads();
  T fro = 0;
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {
    const int i = e % N, j = e / N;
    const T v = A[i + j * ld] * down;
    A[i + j * ld] = v;
    fro += v * v;
  }
  fro = warp_sum(fro);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = fro;
  __syncthreads();
  if (threadIdx.x == 0) {
    T f = 0;
    for (int w = 0; w < kWarpsPerBlock; ++w) f += red[w];
    thr_sh = (T)(PsdEps<T>::v) * sqrt(f);
  }
  __syncthreads();
  const T thr = thr_sh;

  // ---- cyclic Jacobi, round-robin ordering ----
  const int Ne = (N + 1) & ~1;
  const int npairs = Ne / 2;
  int sweep = 0;
  bool converged = false;
  for (; sweep < max_sweeps; ++sweep) {
    if (threadIdx.x == 0) rotated = 0;
    __syncthreads();
    for (int r = 0; r < Ne - 1; ++r) {
      // rotation parameters of this round
      for (int k = threadIdx.x; k < npairs; k += blockDim.x) {
        int p, q;
        rr_pair(Ne, r, k, p, q);
        T c = T(1), sn = T(0);
        if (q < N) {
          const T apq = A[p + q * ld];
          if (tabs(apq) > thr) {
            sym_schur(A[p + p * ld], A[q + q * ld], apq, c, sn);
            rotated = 1;
          }
        }
        cs[2 * k] = c;
        cs[2 * k + 1] = sn;
        pq[2 * k] = p;          // the pairing is computed once per round (integer modulo is expensive)
        pq[2 * k + 1] = q;
      }
      __syncthreads();
      // columns p,q of A and V:  [ap aq] <- [ap aq] * [c s; -s c]
      for (int e = threadIdx.x; e < npairs * N; e += blockDim.x) {
        const int k = e / N, i = e - k * N;
        const T sn = cs[2 * k + 1];
        if (sn == T(0)) continue;
        const T c = cs[2 * k];
        const int p = pq[2 * k], q = pq[2 * k + 1];
        const T aip = A[i + p * ld], aiq = A[i + q * ld];
        A[i + p * ld] = c * aip - sn * aiq;
        A[i + q * ld] = sn * aip + c * aiq;
        const T vip = V[i + p * ld], viq = V[i + q * ld];
        V[i + p * ld] = c * vip - sn * viq;
        V[i + q * ld] = sn * vip + c * viq;
      }
      __syncthreads();
      // rows p,q of A
      for (int e = threadIdx.x; e < npairs * N; e += blockDim.x) {
        const int k = e / N, j = e - k * N;
        const T sn = cs[2 * k + 1];
        if (sn == T(0)) continue;
        const T c = cs[2 * k];
        const int p = pq[2 * k], q = pq[2 * k + 1];
        const T apj = A[p + j * ld], aqj = A[q + j * ld];
        A[p + j * ld] = c * apj - sn * aqj;
        A[q + j * ld] = sn * apj + c * aqj;
      }
      __syncthreads();
    }
    if (!rotated) { converged = true; break; }
    __syncthreads();
  }
  if (!converged && threadIdx.x == 0 && fail_flag) atomicAdd(fail_flag, 1);

  if (mode == 2) {
    T* Q = eig.Q + eig.q_off[blockIdx.x];
    T* lam = eig.lam + eig.lam_off[blockIdx.x];
    const T band = (T)(64.0 * PsdEps<T>::v) * (T(1) + mx_in);
    bool kink = false;
    for (int e = threadIdx.x; e < N * N; e += blockDim.x) {
      const int i = e % N, k = e / N;
      Q[e] = V[i + k * ld];
      if (i == 0) {
        const T l = A[k + k * ld] * up;
        lam[k] = l;
        kink = kink || tabs(l) <= band;
      }
    }
    if (__syncthreads_or(kink) && threadIdx.x == 0) atomicAdd(eig.kinks, 1);
    return;
  }

  if (mode == 1) {
    if (!converged) {
      if (threadIdx.x == 0) lam_max[blockIdx.x] = T(INFINITY);
      return;
    }
    T mx = -INFINITY;
    for (int i = threadIdx.x; i < N; i += blockDim.x) mx = fmax(mx, A[i + i * ld]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
      T f = red[0];
      for (int w = 1; w < kWarpsPerBlock; ++w) f = fmax(f, red[w]);
      lam_max[blockIdx.x] = f * up;
    }
    return;
  }
  // ---- V <- V * diag(sqrt(max(lambda,0))) ; X+ = V V' (rank_k_update!, convexset.jl:243-263) ----
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {
    const int i = e % N, k = e / N;
    const T lam = A[k + k * ld];
    V[i + k * ld] *= (lam > T(0)) ? sqrt(lam) : T(0);
  }
  __syncthreads();
  if (d.triangle == 2) {
    // X+ = A+ + i B+ from the projected embedding P = V V':  A+ = (P11 + P22) / 2,  B+ = (P21 - P12) / 2
    const int Nc = N >> 1;
    const int tri = Nc * (Nc + 1) / 2;
    for (int e = threadIdx.x; e < Nc * Nc; e += blockDim.x) {
      const bool imag = e >= tri;
      const int ee = imag ? e - tri : e;
      int i, j;
      if (!imag) {          // (i, j), i <= j, of the triangle
        j = (int)((sqrt(8.0 * (double)ee + 1.0) - 1.0) * 0.5);
        while ((long long)(j + 1) * (j + 2) / 2 <= ee) ++j;
        while ((long long)j * (j + 1) / 2 > ee) --j;
        i = ee - j * (j + 1) / 2;
      } else {              // (i, j), i < j, of the strict triangle: ee = j (j - 1) / 2 + i
        j = (int)((sqrt(8.0 * (double)ee + 1.0) + 1.0) * 0.5);
        while ((long long)j * (j + 1) / 2 <= ee) ++j;
        while ((long long)j * (j - 1) / 2 > ee) --j;
        i = ee - j * (j - 1) / 2;
      }
      T acc = 0;
      if (!imag) {
        for (int k = 0; k < N; ++k) acc += V[i + k * ld] * V[j + k * ld] + V[Nc + i + k * ld] * V[Nc + j + k * ld];
        acc *= T(0.5);
        s[d.off + e] = ((i == j) ? acc : sqrt2 * acc) * up;
      } else {
        for (int k = 0; k < N; ++k) acc += V[Nc + i + k * ld] * V[j + k * ld] - V[i + k * ld] * V[Nc + j + k * ld];
        s[d.off + e] = sqrt2 * T(0.5) * acc * up;
      }
    }
  } else if (d.triangle) {
    const int tri = N * (N + 1) / 2;
    for (int e = threadIdx.x; e < tri; e += blockDim.x) {
      // invert e -> (i, j), i <= j
      int j = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
      while ((long long)(j + 1) * (j + 2) / 2 <= e) ++j;
      while ((long long)j * (j + 1) / 2 > e) --j;
      const int i = e - j * (j + 1) / 2;
      T acc = 0;
      for (int k = 0; k < N; ++k) acc += V[i + k * ld] * V[j + k * ld];
      s[d.off + e] = ((i == j) ? acc : sqrt2 * acc) * up;
    }
  } else {
    for (int e = threadIdx.x; e < N * N; e += blockDim.x) {
      const int i = e % N, j = e / N;
      const int a = i < j ? i : j, b = i < j ? j : i;
      T acc = 0;
      for (int k = 0; k < N; ++k) acc += V[a + k * ld] * V[b + k * ld];
      s[d.off + e] = acc * up;
    }
  }
}

// ---------------------------------------------------------------------------
// Large cones: matrix + eigenvectors in global memory, one kernel triple per round.
// ---------------------------------------------------------------------------
// Entries a large cone stores: N (N + 1) / 2 (triangle), N^2 (square), Nc^2 (Hermitian, N = 2 Nc).
__host__ __device__ inline long long psd_cone_dim(const PsdConeDesc& d) {
  return d.triangle == 1 ? (long long)d.N * (d.N + 1) / 2 : (d.triangle == 2 ? (long long)(d.N / 2) * (d.N / 2) : (long long)d.N * d.N);
}

// *mx_bits = max(*mx_bits, max |x[0..dim)|) as the bit pattern of a non-negative double (ordered like the value; a NaN
// orders above inf).  *mx_bits must be 0 before the first block runs.
template <typename T>
__global__ void __launch_bounds__(kBlock) psd_cone_max_kernel(const T* __restrict__ x, long long dim, unsigned long long* __restrict__ mx_bits) {
  __shared__ double red[kWarpsPerBlock];
  double mx = 0.0;
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < dim; k += (long long)gridDim.x * blockDim.x) {
    const double v = fabs((double)x[k]);
    mx = (v > mx || v != v) ? v : mx;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double w = __shfl_xor_sync(0xffffffffu, mx, o);
    mx = (w > mx || w != w) ? w : mx;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long b = 0;
    for (int w = 0; w < kWarpsPerBlock; ++w) b = max(b, (unsigned long long)__double_as_longlong(red[w]));
    atomicMax(mx_bits, b);
  }
}

// A = mat(x) 2^-pe, V = I, partial sums of |A|_F^2.  pe (even) is the exponent of the power of two nearest max |x|
// (psd_cone_max_kernel): the scaling is exact, the projection is positively homogeneous, so the eigensolvers and the
// Newton-Schulz iteration work on a matrix of norm ~1 whatever the scale of x; *up = 2^pe undoes it on the output
// (psd_unscale_kernel).  A square cone is symmetrized as project! does, or with upper = 1 reflected from its upper
// triangle as the certificate reads it (see psd_small_kernel).
template <typename T>
__global__ void __launch_bounds__(kBlock) psd_large_load_kernel(PsdConeDesc d, int upper, const T* __restrict__ ws, T* __restrict__ A,
                                                                T* __restrict__ V, T* __restrict__ fro_partials,
                                                                const unsigned long long* __restrict__ mx_bits, double* __restrict__ up) {
  const int N = d.N;
  const T* x = ws + d.off;
  const T inv_sqrt2 = T(0.70710678118654752440);
  const double mxv = __longlong_as_double((long long)*mx_bits);
  const int pe = (mxv == mxv) ? (pow2_exponent((T)mxv) & ~1) : 0;
  const T down = (T)ldexp(1.0, -pe);
  if (blockIdx.x == 0 && threadIdx.x == 0) *up = ldexp(1.0, pe);
  T fro = 0;
  const long long total = (long long)N * N;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % N), j = (int)(e / N);
    T v;
    if (d.triangle == 2) {
      v = hermitian_embedding_entry(x, N >> 1, i, j);
    } else if (d.triangle) {
      const int a = i < j ? i : j, b = i < j ? j : i;
      v = x[svec_pos(a, b)];
      if (a != b) v *= inv_sqrt2;
    } else if (upper) {
      const int a = i < j ? i : j, b = i < j ? j : i;
      v = x[(long long)b * N + a];
    } else {
      v = (x[(long long)j * N + i] + x[(long long)i * N + j]) / T(2);
    }
    v *= down;
    A[e] = v;
    V[e] = (i == j) ? T(1) : T(0);
    fro += v * v;
  }
  __shared__ T red[kWarpsPerBlock];
  fro = warp_sum(fro);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = fro;
  __syncthreads();
  if (threadIdx.x == 0) {
    T f = 0;
    for (int w = 0; w < kWarpsPerBlock; ++w) f += red[w];
    fro_partials[blockIdx.x] = f;
  }
}

// thr = eps * sqrt(sum partials); rotated flag reset
template <typename T>
__global__ void psd_large_thr_kernel(const T* __restrict__ fro_partials, int nparts, T* __restrict__ thr, int* __restrict__ rotated) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    T f = 0;
    for (int i = 0; i < nparts; ++i) f += fro_partials[i];
    *thr = (T)(PsdEps<T>::v) * sqrt(f);
    *rotated = 0;
  }
}

// s[0..dim) *= 2^pe: the projection of the prescaled matrix back to the scale of the input
template <typename T>
__global__ void __launch_bounds__(kBlock) psd_unscale_kernel(T* __restrict__ s, long long dim, const double* __restrict__ up) {
  const double f = *up;
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < dim; k += (long long)gridDim.x * blockDim.x)
    s[k] = (T)((double)s[k] * f);
}

// ---------------------------------------------------------------------------
// Large cones, block Jacobi (two-sided, block size 32): per round the Nb/2 disjoint block
// pairs (I,J) of the round-robin ordering are handled in three launches
//   1. bj_pivot_kernel : one CTA per pair diagonalises its 64x64 pivot [A_II A_IJ; A_JI A_JJ]
//                        in shared memory (<= 2 cyclic Jacobi sweeps) and stores R (64x64)
//   2. bj_cols_kernel  : A[:, I|J] <- A[:, I|J] R  and  V[:, I|J] <- V[:, I|J] R   (64x64x64 tiles)
//   3. bj_rows_kernel  : A[I|J, :] <- R' A[I|J, :]
// so the O(N^3) work is GEMM-shaped and L2-resident; pairs whose pivot is already diagonal
// (to eps |A|_F) are skipped, which is what makes warm starts cheap.
// ---------------------------------------------------------------------------
constexpr int kBjB = 32;          // block size
constexpr int kBjP = 2 * kBjB;    // pivot size

__device__ __forceinline__ int bj_col(int I, int J, int k) { return (k < kBjB) ? I * kBjB + k : J * kBjB + (k - kBjB); }

template <typename T>
__global__ void __launch_bounds__(512) bj_pivot_kernel(int N, int Nb, int r, const T* __restrict__ A, const T* __restrict__ thr_p,
                                                          T* __restrict__ Rbuf, int* __restrict__ active, int* __restrict__ rotated,
                                                          int inner_sweeps) {
  extern __shared__ unsigned char smem_raw[];
  constexpr int P = kBjP, ld = P + 1;
  T* Sa = reinterpret_cast<T*>(smem_raw);
  T* Sv = Sa + ld * P;
  T* cs = Sv + ld * P;
  __shared__ int any_big, rot_flag, round_rot[2];
  __shared__ int pq[kBjP];
  const int k = blockIdx.x;
  int I, J;
  rr_pair(Nb, r, k, I, J);
  const T thr = *thr_p;
  if (threadIdx.x == 0) { any_big = 0; }
  __syncthreads();
  for (int e = threadIdx.x; e < P * P; e += blockDim.x) {
    const int i = e % P, j = e / P;
    const int gi = bj_col(I, J, i), gj = bj_col(I, J, j);
    T v = T(0);
    if (gi < N && gj < N) v = A[gi + (long long)gj * N];
    Sa[i + j * ld] = v;
    Sv[i + j * ld] = (i == j) ? T(1) : T(0);
    if (i != j && tabs(v) > T(8) * thr) any_big = 1;   // activity threshold above the GEMM-update noise floor
  }
  __syncthreads();
  if (!any_big) {
    if (threadIdx.x == 0) active[k] = 0;
    return;
  }
  // symmetrise the pivot copy (the two triangles of A drift by rounding)
  for (int e = threadIdx.x; e < P * P; e += blockDim.x) {
    const int i = e % P, j = e / P;
    if (i < j) {
      const T v = T(0.5) * (Sa[i + j * ld] + Sa[j + i * ld]);
      Sa[i + j * ld] = v;
      Sa[j + i * ld] = v;
    }
  }
  __syncthreads();
  const int npairs = P / 2;
  for (int sweep = 0; sweep < inner_sweeps; ++sweep) {
    if (threadIdx.x == 0) rot_flag = 0;
    __syncthreads();
    for (int rr = 0; rr < P - 1; ++rr) {
      const int f = rr & 1;   // alternating flag: its reset two rounds later cannot race with this round's reads
      if (threadIdx.x == 0) round_rot[f] = 0;
      __syncthreads();
      for (int kk = threadIdx.x; kk < npairs; kk += blockDim.x) {
        int p, q;
        rr_pair(P, rr, kk, p, q);
        T c = T(1), sn = T(0);
        const T apq = Sa[p + q * ld];
        if (tabs(apq) > thr) {
          sym_schur(Sa[p + p * ld], Sa[q + q * ld], apq, c, sn);
          rot_flag = 1;
          round_rot[f] = 1;
        }
        cs[2 * kk] = c;
        cs[2 * kk + 1] = sn;
        pq[2 * kk] = p;
        pq[2 * kk + 1] = q;
      }
      __syncthreads();
      if (!round_rot[f]) continue;   // nothing to rotate in this round (block-uniform)
      for (int e = threadIdx.x; e < npairs * P; e += blockDim.x) {
        const int kk = e / P, i = e % P;
        const T sn = cs[2 * kk + 1];
        if (sn == T(0)) continue;
        const T c = cs[2 * kk];
        const int p = pq[2 * kk], q = pq[2 * kk + 1];
        const T aip = Sa[i + p * ld], aiq = Sa[i + q * ld];
        Sa[i + p * ld] = c * aip - sn * aiq;
        Sa[i + q * ld] = sn * aip + c * aiq;
        const T vip = Sv[i + p * ld], viq = Sv[i + q * ld];
        Sv[i + p * ld] = c * vip - sn * viq;
        Sv[i + q * ld] = sn * vip + c * viq;
      }
      __syncthreads();
      for (int e = threadIdx.x; e < npairs * P; e += blockDim.x) {
        const int kk = e / P, j = e % P;
        const T sn = cs[2 * kk + 1];
        if (sn == T(0)) continue;
        const T c = cs[2 * kk];
        const int p = pq[2 * kk], q = pq[2 * kk + 1];
        const T apj = Sa[p + j * ld], aqj = Sa[q + j * ld];
        Sa[p + j * ld] = c * apj - sn * aqj;
        Sa[q + j * ld] = sn * apj + c * aqj;
      }
      __syncthreads();
    }
    if (!rot_flag) break;
    __syncthreads();
  }
  T* R = Rbuf + (size_t)k * P * P;
  for (int e = threadIdx.x; e < P * P; e += blockDim.x) R[e] = Sv[(e % P) + (e / P) * ld];
  if (threadIdx.x == 0) { active[k] = 1; *rotated = 1; }
}

// ---- GEMM-shaped block updates -------------------------------------------------------------
// 64 threads own one 64x64 output tile with an 8x8 register micro-tile each (64 FP64 accumulators,
// 8 LDS.128 per 64 DFMA => FP64-pipe bound instead of shared-memory bound); a 256-thread CTA handles
// four tiles that share the same 64x64 rotation R (stored transposed in shared memory).
constexpr int kBjLd = kBjP + 2;        // even leading dimension: 16-byte aligned columns for LDS.128
constexpr int kBjTilesPerCta = 4;

template <typename T>
__device__ __forceinline__ void bj_load8(const T* p, T (&v)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = p[k];
}

// X[:, I|J] <- X[:, I|J] * R  for X = A (blockIdx.z = 0) and V (blockIdx.z = 1), 4 row tiles per CTA
template <typename T>
__global__ void __launch_bounds__(kBlock, 1) bj_cols_kernel(int N, int Nb, int r, T* __restrict__ A, T* __restrict__ V,
                                                            const T* __restrict__ Rbuf, const int* __restrict__ active) {
  const int k = blockIdx.y;
  if (!active[k]) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int P = kBjP, ld = kBjLd;
  T* Rt = reinterpret_cast<T*>(smem_raw);            // Rt[kk * P + j] = R[kk][j]
  T* S = Rt + P * P;                                 // 4 tiles: S[g][i + kk * ld]
  T* X = (blockIdx.z == 0) ? A : V;
  int I, J;
  rr_pair(Nb, r, k, I, J);
  const T* R = Rbuf + (size_t)k * P * P;             // column-major R[i + j * P]
  for (int e = threadIdx.x; e < P * P; e += blockDim.x) {
    const int i = e % P, j = e / P;
    Rt[i * P + j] = R[e];
  }
  const int row_base = blockIdx.x * (P * kBjTilesPerCta);
  for (int e = threadIdx.x; e < kBjTilesPerCta * P * P; e += blockDim.x) {
    const int g = e / (P * P), rem = e % (P * P);
    const int i = rem % P, j = rem / P;
    const int gi = row_base + g * P + i, gj = bj_col(I, J, j);
    S[g * (ld * P) + i + j * ld] = (gi < N && gj < N) ? X[gi + (long long)gj * N] : T(0);
  }
  __syncthreads();
  const int g = threadIdx.x / 64, t = threadIdx.x % 64;
  const int ti = (t % 8) * 8, tj = (t / 8) * 8;
  const T* Sg = S + g * (ld * P);
  T acc[8][8];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[a][b] = T(0);
#pragma unroll 2
  for (int kk = 0; kk < P; ++kk) {
    T sv[8], rv[8];
    bj_load8(Sg + ti + kk * ld, sv);
    bj_load8(Rt + kk * P + tj, rv);
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
      for (int b = 0; b < 8; ++b) acc[a][b] += sv[a] * rv[b];
  }
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const int gj = bj_col(I, J, tj + b);
    if (gj >= N) continue;
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      const int gi = row_base + g * P + ti + a;
      if (gi < N) X[gi + (long long)gj * N] = acc[a][b];
    }
  }
}

// A[I|J, :] <- R' * A[I|J, :], 4 column tiles per CTA
template <typename T>
__global__ void __launch_bounds__(kBlock, 1) bj_rows_kernel(int N, int Nb, int r, T* __restrict__ A, const T* __restrict__ Rbuf,
                                                            const int* __restrict__ active) {
  const int k = blockIdx.y;
  if (!active[k]) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int P = kBjP, ld = kBjLd;
  T* Rc = reinterpret_cast<T*>(smem_raw);            // Rc[kk * P + i] = R[kk][i]  (row kk of R: contiguous in i)
  T* Tt = Rc + P * P;                                // 4 tiles: Tt[g][kk * ld + j] = A[pivot row kk][col j]
  int I, J;
  rr_pair(Nb, r, k, I, J);
  const T* R = Rbuf + (size_t)k * P * P;
  for (int e = threadIdx.x; e < P * P; e += blockDim.x) {
    const int i = e % P, j = e / P;                  // R[i + j*P] = R[i][j]
    Rc[i * P + j] = R[e];
  }
  const int col_base = blockIdx.x * (P * kBjTilesPerCta);
  for (int e = threadIdx.x; e < kBjTilesPerCta * P * P; e += blockDim.x) {
    const int g = e / (P * P), rem = e % (P * P);
    const int i = rem % P, j = rem / P;              // i: pivot row (contiguous in memory), j: column in tile
    const int gi = bj_col(I, J, i), gj = col_base + g * P + j;
    Tt[g * (ld * P) + i * ld + j] = (gi < N && gj < N) ? A[gi + (long long)gj * N] : T(0);
  }
  __syncthreads();
  const int g = threadIdx.x / 64, t = threadIdx.x % 64;
  const int ti = (t % 8) * 8, tj = (t / 8) * 8;       // out[ti..ti+7][tj..tj+7] = sum_kk R[kk][ti+a] * T[kk][tj+b]
  const T* Tg = Tt + g * (ld * P);
  T acc[8][8];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[a][b] = T(0);
#pragma unroll 2
  for (int kk = 0; kk < P; ++kk) {
    T rv[8], tv[8];
    bj_load8(Rc + kk * P + ti, rv);
    bj_load8(Tg + kk * ld + tj, tv);
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
      for (int b = 0; b < 8; ++b) acc[a][b] += rv[a] * tv[b];
  }
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const int gj = col_base + g * P + tj + b;
    if (gj >= N) continue;
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      const int gi = bj_col(I, J, ti + a);
      if (gi < N) A[gi + (long long)gj * N] = acc[a][b];
    }
  }
}

// C (N x N) = op(A) * B, column-major, op(A) = A or A'; 128x128 CTA tile, 8x8 register micro-tiles,
// K in chunks of 16 through shared memory.  Used for the warm start  A <- V0' (X V0).
template <typename T, bool TRANSA>
__global__ void __launch_bounds__(kBlock, 1) bj_gemm_kernel(int N, const T* __restrict__ A, const T* __restrict__ B,
                                                            T* __restrict__ C) {
  constexpr int TM = 128, TK = 16, LDS_ = TM + 2;
  __shared__ __align__(16) T As[TK][LDS_];   // As[kk][i] = op(A)[row0 + i][k0 + kk]
  __shared__ __align__(16) T Bs[TK][LDS_];   // Bs[kk][j] = B[k0 + kk][col0 + j]
  const int row0 = blockIdx.x * TM, col0 = blockIdx.y * TM;
  const int ti = (threadIdx.x % 16) * 8, tj = (threadIdx.x / 16) * 8;
  T acc[8][8];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[a][b] = T(0);
  for (int k0 = 0; k0 < N; k0 += TK) {
    for (int e = threadIdx.x; e < TK * TM; e += blockDim.x) {
      int kk, i;
      if (TRANSA) { kk = e % TK; i = e / TK; } else { i = e % TM; kk = e / TM; }
      const int gi = row0 + i, gk = k0 + kk;
      T v = T(0);
      if (gi < N && gk < N) v = TRANSA ? A[gk + (long long)gi * N] : A[gi + (long long)gk * N];
      As[kk][i] = v;
    }
    for (int e = threadIdx.x; e < TK * TM; e += blockDim.x) {
      const int kk = e % TK, j = e / TK;
      const int gk = k0 + kk, gj = col0 + j;
      Bs[kk][j] = (gk < N && gj < N) ? B[gk + (long long)gj * N] : T(0);
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < TK; ++kk) {
      T av[8], bv[8];
      bj_load8(&As[kk][ti], av);
      bj_load8(&Bs[kk][tj], bv);
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) acc[a][b] += av[a] * bv[b];
    }
    __syncthreads();
  }
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const int gj = col0 + tj + b;
    if (gj >= N) continue;
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      const int gi = row0 + ti + a;
      if (gi < N) C[gi + (long long)gj * N] = acc[a][b];
    }
  }
}

// V[:,k] *= sqrt(max(lambda_k, 0))
template <typename T>
__global__ void __launch_bounds__(kBlock) psd_large_scale_kernel(int N, const T* __restrict__ A, T* __restrict__ V) {
  const long long total = (long long)N * N;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(e / N);
    const T lam = A[k + (long long)k * N];
    V[e] *= (lam > T(0)) ? sqrt(lam) : T(0);
  }
}

// out = svec / square of (V V') upper triangle, 32x32 output tiles, K-tiles of 32 through shared memory
template <typename T>
__global__ void __launch_bounds__(256) psd_large_syrk_kernel(PsdConeDesc d, const T* __restrict__ V, T* __restrict__ s) {
  const int N = d.N;
  const int bi = blockIdx.x, bj = blockIdx.y;
  if (bi > bj) return;  // upper triangle of tiles
  __shared__ T Vi[32][33];
  __shared__ T Vj[32][33];
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;  // ty in [0, 8)
  T acc[4] = {0, 0, 0, 0};
  for (int k0 = 0; k0 < N; k0 += 32) {
    for (int rr = ty; rr < 32; rr += 8) {   // rr: k within tile, tx: row within tile (coalesced along rows)
      const int k = k0 + rr;
      const int gi = bi * 32 + tx, gj = bj * 32 + tx;
      Vi[rr][tx] = (k < N && gi < N) ? V[gi + (long long)k * N] : T(0);
      Vj[rr][tx] = (k < N && gj < N) ? V[gj + (long long)k * N] : T(0);
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const T vi = Vi[k][tx];
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] += vi * Vj[k][ty + 8 * u];
    }
    __syncthreads();
  }
  const T sqrt2 = T(1.41421356237309504880);
  const int i = bi * 32 + tx;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int j = bj * 32 + ty + 8 * u;
    if (i < N && j < N && i <= j) {
      if (d.triangle) {
        s[d.off + svec_pos(i, j)] = (i == j) ? acc[u] : sqrt2 * acc[u];
      } else {
        s[d.off + (long long)j * N + i] = acc[u];
        s[d.off + (long long)i * N + j] = acc[u];   // mirror, convexset.jl:316-318
      }
    }
  }
}

template <typename T>
__global__ void psd_large_lammax_kernel(int N, const T* __restrict__ A, const double* __restrict__ up, T* __restrict__ out) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    T mx = -INFINITY;
    for (int i = 0; i < N; ++i) mx = fmax(mx, A[i + (long long)i * N]);
    *out = (T)((double)mx * *up);
  }
}

}  // namespace cosmo
#include "psd_tc.cuh"
namespace cosmo {

// ---------------------------------------------------------------------------
// Host-side batch object
// ---------------------------------------------------------------------------
template <typename T>
struct PsdBatch {
  std::vector<PsdConeDesc> small_h, large_h;
  DevBuf<PsdConeDesc> small_d;
  DevBuf<T> lam_small_d;
  DevBuf<int> fail_d;
  int small_maxN = 0;
  // large-cone workspace (sized for the largest cone, cones processed one after another)
  int large_maxN = 0;
  DevBuf<T> A_d, V_d, fro_d, thr_d, lam_large_d;
  DevBuf<int> rot_d;
  PinnedBuf<int> rot_h;
  DevBuf<unsigned long long> mx_d;   // max |entry| of the cone being projected (psd_cone_max_kernel)
  DevBuf<double> up_d;               // 2^pe: the prescaling of that cone (psd_large_load_kernel)
  // warm start across ADMM iterations (single large cone): eigenvectors of the previous projection
  DevBuf<T> Vw_d, T_d;
  bool warm_valid = false;
  int warm_N = 0;
  long long warm_count = 0;
  int last_sweeps = 0;
  PsdTc<T> tc_;          // tensor-core projection (psd_tc.cuh): Newton-Schulz on int8-sliced wgmma products
  bool tc_enabled = PsdTc<T>::enabled();
  long long tc_projections = 0, tc_fallbacks = 0;
  DevBuf<T> R_d;         // npairs * 64 * 64 pivot rotations
  DevBuf<int> act_d;     // per pair: pivot needed work this round
  std::vector<T> lam_host;
  std::vector<int> small_idx, large_idx;   // position of each small / large cone among all PSD cones (set order)
  std::vector<double> lam_all;
  int cert_unconverged = 0;                // cones whose eigensolver missed max_sweeps in the last lambda_max call

  bool empty() const { return small_h.empty() && large_h.empty(); }

  void init(const std::vector<PsdConeDesc>& descs, cudaStream_t st) {
    for (size_t k = 0; k < descs.size(); ++k) {
      const bool small = descs[k].N <= kPsdSmallMax;
      (small ? small_h : large_h).push_back(descs[k]);
      (small ? small_idx : large_idx).push_back((int)k);
    }
    if (!small_h.empty()) {
      for (const auto& d : small_h) small_maxN = std::max(small_maxN, d.N);
      small_d.upload(small_h, st);
      lam_small_d.alloc(small_h.size(), false);
      // the attribute belongs to the function on the device, not to this engine: always raise it to the worst case
      // of kPsdSmallMax, or a second engine with smaller cones would lower the limit under a live one
      const size_t ld_max = (size_t)(kPsdSmallMax | 1);
      const size_t smem = (2 * ld_max * kPsdSmallMax + 2 * (size_t)(kPsdSmallMax / 2 + 2)) * sizeof(T);
      CUDA_TRY(cudaFuncSetAttribute(psd_small_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    fail_d.alloc(1, false);
    CUDA_TRY(cudaMemsetAsync(fail_d.p, 0, sizeof(int), st));
    if (!large_h.empty()) {
      for (const auto& d : large_h) large_maxN = std::max(large_maxN, d.N);
      const size_t nn = (size_t)large_maxN * large_maxN;
      A_d.alloc(nn, false); V_d.alloc(nn, false); fro_d.alloc(kMaxGrid, false);
      thr_d.alloc(1, false); lam_large_d.alloc(large_h.size(), false); rot_d.alloc(1, false); rot_h.alloc(1);
      mx_d.alloc(1, false); up_d.alloc(1, false);
      if (large_h.size() == 1) { Vw_d.alloc(nn, false); T_d.alloc(nn, false); }
      int Nb = (large_maxN + kBjB - 1) / kBjB;
      if (Nb & 1) ++Nb;
      R_d.alloc((size_t)(Nb / 2) * kBjP * kBjP, false);
      act_d.alloc(Nb / 2, false);
      const int smem_pivot = (int)((2 * (size_t)(kBjP + 1) * kBjP + kBjP + 2) * sizeof(T));
      const int smem_upd = (int)(((size_t)kBjP * kBjP + (size_t)kBjTilesPerCta * kBjLd * kBjP) * sizeof(T));
      CUDA_TRY(cudaFuncSetAttribute(bj_pivot_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_pivot));
      CUDA_TRY(cudaFuncSetAttribute(bj_cols_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_upd));
      CUDA_TRY(cudaFuncSetAttribute(bj_rows_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_upd));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  size_t small_smem() const {
    const size_t ld = (size_t)(small_maxN | 1);
    return (2 * ld * small_maxN + 2 * (size_t)(small_maxN / 2 + 2)) * sizeof(T);
  }
  void reset_warm_start() { warm_valid = false; warm_count = 0; }

  // A_d = mat(ws[cone]) 2^-pe, V_d = I, fro_d = partial sums of |A_d|_F^2 (g of them), up_d = 2^pe
  // upper: reflect a square cone from its upper triangle (the certificate) instead of symmetrizing it (the projection)
  void load_large(const PsdConeDesc& d, const T* ws, cudaStream_t st, long long& launches, bool upper = false) {
    const int N = d.N;
    const int g = (int)std::min<long long>(((long long)N * N + kBlock - 1) / kBlock, kMaxGrid);
    const long long dim = psd_cone_dim(d);
    const int gm = (int)std::min<long long>((dim + kBlock - 1) / kBlock, kMaxGrid);
    CUDA_TRY(cudaMemsetAsync(mx_d.p, 0, sizeof(unsigned long long), st));
    psd_cone_max_kernel<T><<<gm, kBlock, 0, st>>>(ws + d.off, dim, mx_d.p);
    psd_large_load_kernel<T><<<g, kBlock, 0, st>>>(d, upper ? 1 : 0, ws, A_d.p, V_d.p, fro_d.p, mx_d.p, up_d.p);
    launches += 2;
  }
  void unscale_large(const PsdConeDesc& d, T* s, cudaStream_t st, long long& launches) {
    const long long dim = psd_cone_dim(d);
    psd_unscale_kernel<T><<<(int)std::min<long long>((dim + kBlock - 1) / kBlock, kMaxGrid), kBlock, 0, st>>>(s + d.off, dim, up_d.p);
    ++launches;
  }

  // eigen-decompose one large cone into A_d (diagonal = eigenvalues) and V_d (block Jacobi).  certificate: load a
  // square cone from its upper triangle and return false instead of throwing ERR_NUMERICAL when max_sweeps is not enough;
  // no_throw alone: the latter only (the eigenpairs of the projection's matrix, solve_adjoint.cuh).
  bool large_eig(const PsdConeDesc& d, const T* ws, cudaStream_t st, int max_sweeps, long long& launches,
                 bool allow_warm = false, bool certificate = false, bool no_throw = false) {
    const int N = d.N;
    int Nb = (N + kBjB - 1) / kBjB;
    if (Nb & 1) ++Nb;                                 // even number of blocks (zero padding decouples)
    const int npairs = Nb / 2;
    const int g = (int)std::min<long long>(((long long)N * N + kBlock - 1) / kBlock, kMaxGrid);
    load_large(d, ws, st, launches, certificate);
    psd_large_thr_kernel<T><<<1, 32, 0, st>>>(fro_d.p, g, thr_d.p, rot_d.p);
    ++launches;
    // Warm start (ADMM iterates move slowly): rotate X into the eigenbasis of the previous projection,
    // A <- V0' X V0 is then nearly diagonal and a couple of sweeps finish the job; V starts at V0.
    // A cold start every 16th call bounds the drift of V's orthogonality.
    const bool warm = allow_warm && Vw_d.p && warm_valid && warm_N == N && (warm_count % 16 != 0);
    if (warm) {
      dim3 gg((N + 127) / 128, (N + 127) / 128);
      bj_gemm_kernel<T, false><<<gg, kBlock, 0, st>>>(N, A_d.p, Vw_d.p, T_d.p);     // T = X V0
      bj_gemm_kernel<T, true><<<gg, kBlock, 0, st>>>(N, Vw_d.p, T_d.p, A_d.p);      // A = V0' T
      CUDA_TRY(cudaMemcpyAsync(V_d.p, Vw_d.p, (size_t)N * N * sizeof(T), cudaMemcpyDeviceToDevice, st));
      launches += 2;
    }
    const size_t smem_pivot = (2 * (size_t)(kBjP + 1) * kBjP + kBjP + 2) * sizeof(T);
    const size_t smem_upd = ((size_t)kBjP * kBjP + (size_t)kBjTilesPerCta * kBjLd * kBjP) * sizeof(T);
    const int tiles = (N + kBjP * kBjTilesPerCta - 1) / (kBjP * kBjTilesPerCta);
    bool converged = false;
    int sweep = 0;
    for (; sweep < max_sweeps && !converged; ++sweep) {
      for (int r = 0; r < Nb - 1; ++r) {
        bj_pivot_kernel<T><<<npairs, 512, smem_pivot, st>>>(N, Nb, r, A_d.p, thr_d.p, R_d.p, act_d.p, rot_d.p, 1);
        bj_cols_kernel<T><<<dim3(tiles, npairs, 2), kBlock, smem_upd, st>>>(N, Nb, r, A_d.p, V_d.p, R_d.p, act_d.p);
        bj_rows_kernel<T><<<dim3(tiles, npairs, 1), kBlock, smem_upd, st>>>(N, Nb, r, A_d.p, R_d.p, act_d.p);
        launches += 3;
      }
      CUDA_TRY(cudaMemcpyAsync(rot_h.p, rot_d.p, sizeof(int), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaMemsetAsync(rot_d.p, 0, sizeof(int), st));
      CUDA_TRY(cudaStreamSynchronize(st));
      if (rot_h[0] == 0) converged = true;
    }
    last_sweeps = sweep;
    if (getenv("COSMO_B200_PSD_DEBUG")) fprintf(stderr, "[psd] N=%d warm=%d sweeps=%d\n", N, (int)warm, sweep);
    CUDA_TRY(cudaGetLastError());
    if (!converged) {
      if (certificate || no_throw) return false;
      throw EngineError{COSMO_B200_ERR_NUMERICAL, "block Jacobi eigensolver did not converge within psd_max_sweeps"};
    }
    if (allow_warm && Vw_d.p) {
      CUDA_TRY(cudaMemcpyAsync(Vw_d.p, V_d.p, (size_t)N * N * sizeof(T), cudaMemcpyDeviceToDevice, st));
      warm_valid = true;
      warm_N = N;
      ++warm_count;
    }
    return true;
  }

  // s[cone rows] = Pi_PSD(ws[cone rows]) for every PSD cone
  void project(const T* ws, T* s, cudaStream_t st, int max_sweeps, long long& launches) {
    if (empty()) return;
    if (max_sweeps <= 0) max_sweeps = 30;
    if (!small_h.empty()) {
      psd_small_kernel<T><<<(int)small_h.size(), kBlock, small_smem(), st>>>(small_d.p, ws, s, 0, lam_small_d.p, max_sweeps, fail_d.p);
      CUDA_TRY(cudaGetLastError());
      ++launches;
    }
    for (const auto& d : large_h) {
      if (tc_enabled) {
        const int N = d.N;
        const int g = (int)std::min<long long>(((long long)N * N + kBlock - 1) / kBlock, kMaxGrid);
        load_large(d, ws, st, launches);
        if (tc_.project(d, A_d.p, fro_d.p, g, V_d.p, s, st, launches)) {
          unscale_large(d, s, st, launches);
          ++tc_projections;
          continue;
        }
        ++tc_fallbacks;
      }
      large_eig(d, ws, st, max_sweeps, launches, /*allow_warm=*/true);
      const int N = d.N;
      const int g = (int)std::min<long long>(((long long)N * N + kBlock - 1) / kBlock, kMaxGrid);
      psd_large_scale_kernel<T><<<g, kBlock, 0, st>>>(N, A_d.p, V_d.p);
      dim3 gt((N + 31) / 32, (N + 31) / 32);
      if (d.triangle == 2) {
        // Hermitian cone: reconstruct the projected embedding as a square matrix in A_d (its eigenvalues are no longer
        // needed), then read A+ and B+ off its blocks
        const PsdConeDesc sq{0, N, 0};
        psd_large_syrk_kernel<T><<<gt, 256, 0, st>>>(sq, V_d.p, A_d.p);
        psd_embedding_store_kernel<T, T><<<g, kBlock, 0, st>>>(d, A_d.p, s);
        ++launches;
      } else {
        psd_large_syrk_kernel<T><<<gt, 256, 0, st>>>(d, V_d.p, s);
      }
      unscale_large(d, s, st, launches);
      CUDA_TRY(cudaGetLastError());
      launches += 2;
    }
  }

  // true iff lambda_max(mat(v_cone)) < tol for every PSD cone, i.e. -mat(v) + tol I is
  // positive definite (is_pos_def!/is_neg_def!, algebra.jl:226-238; convexset.jl:324-336,415-425)
  bool certificate(const T* v, bool /*negate*/, double tol, cudaStream_t st, int max_sweeps, long long& launches) {
    if (empty()) return true;
    lam_all.resize(small_h.size() + large_h.size());
    lambda_max(v, st, max_sweeps, launches, lam_all.data());
    bool ok = true;
    for (double l : lam_all) if (!(l < tol)) ok = false;
    return ok;
  }

  // lam[k] = lambda_max of the k-th PSD cone (set order) of mat(v), read as the certificate reads it (a square cone
  // from its upper triangle); +inf for a cone whose eigensolver did not converge within max_sweeps (counted in
  // cert_unconverged).  Small cones: psd_small_kernel mode 1; large cones: block Jacobi + psd_large_lammax_kernel.
  void lambda_max(const T* v, cudaStream_t st, int max_sweeps, long long& launches, double* lam) {
    if (max_sweeps <= 0) max_sweeps = 30;
    cert_unconverged = 0;
    if (!small_h.empty()) {
      CUDA_TRY(cudaMemsetAsync(fail_d.p, 0, sizeof(int), st));
      psd_small_kernel<T><<<(int)small_h.size(), kBlock, small_smem(), st>>>(small_d.p, v, nullptr, 1, lam_small_d.p, max_sweeps, fail_d.p);
      CUDA_TRY(cudaGetLastError());
      ++launches;
      lam_host.resize(small_h.size());
      int fails = 0;
      CUDA_TRY(cudaMemcpyAsync(lam_host.data(), lam_small_d.p, small_h.size() * sizeof(T), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaMemcpyAsync(&fails, fail_d.p, sizeof(int), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      for (size_t k = 0; k < small_h.size(); ++k) lam[small_idx[k]] = (double)lam_host[k];
      cert_unconverged += fails;
    }
    for (size_t k = 0; k < large_h.size(); ++k) {
      if (!large_eig(large_h[k], v, st, max_sweeps, launches, /*allow_warm=*/false, /*certificate=*/true)) {
        lam[large_idx[k]] = INFINITY;
        ++cert_unconverged;
        continue;
      }
      psd_large_lammax_kernel<T><<<1, 32, 0, st>>>(large_h[k].N, A_d.p, up_d.p, lam_large_d.p + k);
      ++launches;
      T l;
      CUDA_TRY(cudaMemcpyAsync(&l, lam_large_d.p + k, sizeof(T), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      lam[large_idx[k]] = (double)l;
    }
  }
};

}  // namespace cosmo
