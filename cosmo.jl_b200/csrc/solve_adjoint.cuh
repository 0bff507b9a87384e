// solve_adjoint.cuh -- derivatives of a conic solution through the fixed point of the ADMM iteration
// (cosmo_b200_solve_adjoint, DESIGN.md §3k, and its forward counterpart cosmo_b200_solve_derivative, §3l).
//
// In the engine's scaled coordinates an alpha = 1 step of the iteration is
//   T1(w) = [x~; Pi(w_s) - nu/rho],  [x~; nu] = K^-1 [sigma w_x - q; b - 2 Pi(w_s) + w_s],  K = [P + sigma I, A'; A, -1/rho]
// and its linearisation at the fixed point is M = E K^-1 F + G with E = diag(I, -1/rho), F = diag(sigma I, I - 2 Dpi),
// G = diag(0, Dpi), Dpi = DPi(w_s).  Every factor is symmetric, so
//   (I - M') lam = lam - [sigma a; b + Dpi(lam_s - 2 b)],  [a; b] = K^-1 [lam_x; -lam_s / rho]:
// one plugin solve and one Jacobian application per operator application.  GMRES solves (I - M') lam = gw on the
// device (the small Hessenberg system lives on the host); the gradients follow from [u; v] = K^-1 [lam_x; -lam_s / rho].
//
// The kernels here form the Jacobian data of the point (row flags, SOC norms, the eigenpairs of every PSD cone), apply
// Dpi, run the Krylov vector work and write the gradients.  Every reduction sums fixed-order block partials and every
// count uses integer atomics only, so a call is bitwise reproducible.
#pragma once
#include "common.cuh"
#include "psd.cuh"
#include "vector_kernels.cuh"

namespace cosmo {

// integer counters of a call (deterministic: __syncthreads_count and one integer atomic per block)
enum { SA_CNT_ROWS = 0, SA_CNT_SOC = 1, SA_CNT_PSD = 2, SA_CNT_PSD_UNCONVERGED = 3, SA_CNT_COUNT = 4 };
// flag byte of a Nonnegatives or Box row at w_s: Dpi = 1 strictly inside, else the bound w_s is clamped to
enum : unsigned char { SA_ROW_OUT = 0, SA_ROW_IN = 1, SA_ROW_LOWER = 2, SA_ROW_UPPER = 4 };

// the kink band of a cone: 64 u (1 + |w_s|), u the unit roundoff of T
template <typename T>
__device__ __forceinline__ double sa_kink_band(double w) {
  return 64.0 * PsdEps<T>::v * (1.0 + w);
}

// block-wide count of `pred` added to *cnt with one integer atomic; every thread of the block must call it
__device__ __forceinline__ void sa_count(bool pred, int* cnt) {
  const int c = __syncthreads_count(pred);
  if (threadIdx.x == 0 && c) atomicAdd(cnt, c);
}

// flags of the Nonnegatives and Box rows at w_s (0 on every other row) and the rows near a kink
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_row_flags_kernel(int m, const unsigned char* __restrict__ row_class,
                                                              const T* __restrict__ ws, const T* __restrict__ box_l,
                                                              const T* __restrict__ box_u, unsigned char* __restrict__ flag,
                                                              int* __restrict__ counts) {
  const int stride = gridDim.x * blockDim.x;
  const int rounds = (m + stride - 1) / stride;
  for (int k = 0, r = blockIdx.x * blockDim.x + threadIdx.x; k < rounds; ++k, r += stride) {
    bool kink = false;
    if (r < m) {
      const unsigned char cls = row_class[r];
      unsigned char f = SA_ROW_OUT;
      const double w = (double)ws[r];
      const double band = sa_kink_band<T>(fabs(w));
      if (cls == ROW_NONNEG) {
        f = w > 0.0 ? SA_ROW_IN : SA_ROW_OUT;
        kink = fabs(w) <= band;
      } else if (cls == ROW_BOX) {
        const double l = (double)box_l[r], u = (double)box_u[r];
        f = (w > l && w < u) ? SA_ROW_IN : (w <= l ? SA_ROW_LOWER : SA_ROW_UPPER);
        kink = fabs(w - l) <= band || fabs(w - u) <= band;
      }
      flag[r] = f;
    }
    sa_count(kink, counts + SA_CNT_ROWS);
  }
}

// SOC cones near a kink: | |xbar| - |t| | within the band of the cone
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_soc_kink_kernel(int ncones, const int* __restrict__ soc_off, const T* __restrict__ ws,
                                                             const T* __restrict__ norm, int* __restrict__ counts) {
  const int stride = gridDim.x * blockDim.x;
  const int rounds = (ncones + stride - 1) / stride;
  for (int k = 0, c = blockIdx.x * blockDim.x + threadIdx.x; k < rounds; ++k, c += stride) {
    bool kink = false;
    if (c < ncones) {
      const double t = (double)ws[soc_off[c]], r = (double)norm[c];
      kink = fabs(r - fabs(t)) <= sa_kink_band<T>(fmax(fabs(t), r));
    }
    sa_count(kink, counts + SA_CNT_SOC);
  }
}

// The SOC terms are formed from dhat = xbar'hbar / r, summed with xbar scaled by 2^-e, e = pow2_exponent(r) (exact):
// every scaled entry is below 1 in magnitude, so the sum neither overflows nor underflows where h does not, whatever
// the scale of w_s (an unscaled xbar'hbar overflows at |w_s| |h| > 2^1024 and flushes to 0 below 2^-1074)
__device__ __forceinline__ int sa_soc_exponent(double r) { return pow2_exponent<double>(r); }

// 2^-e xbar'h per chunk of a SOC tail (fixed-order block tree), the partials the next kernel folds per cone; the cone
// of chunk c is the last k with cone_chunk_ptr[k] <= c
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_soc_dot_chunk_kernel(const T* __restrict__ ws, const T* __restrict__ h,
                                                                  const int* __restrict__ chunk_start,
                                                                  const int* __restrict__ chunk_len,
                                                                  const int* __restrict__ cone_chunk_ptr, int ncones,
                                                                  const T* __restrict__ norm, double* __restrict__ chunk_dot) {
  __shared__ double sm[kWarpsPerBlock];
  const int c = blockIdx.x;
  const int start = chunk_start[c], len = chunk_len[c];
  int lo = 0, hi = ncones - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cone_chunk_ptr[mid] <= c) lo = mid;
    else hi = mid - 1;
  }
  const double down = ldexp(1.0, -sa_soc_exponent((double)norm[lo]));
  double acc = 0.0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) acc += ((double)ws[start + i] * down) * (double)h[start + i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = sm[0];
    for (int w = 1; w < kWarpsPerBlock; ++w) v += sm[w];
    chunk_dot[c] = v;
  }
}

// dhat[k] = (sum of cone k's chunk partials in chunk order) / (2^-e r), 0 when r = 0 (no branch reads it then)
template <typename T>
__global__ void sa_soc_dot_final_kernel(const double* __restrict__ chunk_dot, const int* __restrict__ cone_chunk_ptr, int ncones,
                                        const T* __restrict__ norm, double* __restrict__ dhat) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ncones) return;
  double v = 0.0;
  for (int c = cone_chunk_ptr[k]; c < cone_chunk_ptr[k + 1]; ++c) v += chunk_dot[c];
  const double r = (double)norm[k];
  const double rs = ldexp(r, -sa_soc_exponent(r));
  dhat[k] = rs > 0.0 ? v / rs : 0.0;
}

// out = Dpi h on every row outside the PSD and custom cones (those are written by the PSD kernels and the custom cones'
// Jacobian hooks):
//   ZeroSet 0;  Nonnegatives, Box: h strictly inside, 0 outside;
//   SOC (t, xbar), r = |xbar|, dhat = xbar'hbar / r: h if r <= t, 0 if r <= -t, else
//     1/2 [h_t + dhat ;  (xbar / r) h_t + (1 + t/r) hbar - (t/r) (xbar / r) dhat]
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_dpi_rows_kernel(int m, const unsigned char* __restrict__ row_class,
                                                             const int* __restrict__ row_cone, const unsigned char* __restrict__ flag,
                                                             const int* __restrict__ soc_off, const T* __restrict__ ws,
                                                             const T* __restrict__ soc_r, const double* __restrict__ soc_dhat,
                                                             const T* __restrict__ h, T* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const unsigned char cls = row_class[i];
    if (cls == ROW_PSD || cls == ROW_CUSTOM) continue;
    T v = T(0);
    if (cls == ROW_NONNEG || cls == ROW_BOX) {
      v = flag[i] == SA_ROW_IN ? h[i] : T(0);
    } else if (cls == ROW_SOC) {
      const int k = row_cone[i];
      const int off = soc_off[k];
      const double t = (double)ws[off], r = (double)soc_r[k];
      if (r <= t) {
        v = h[i];
      } else if (r > -t) {
        const double d = soc_dhat[k];
        if (i == off) {
          v = (T)(0.5 * ((double)h[off] + d));
        } else {
          const double xr = (double)ws[i] / r, tr = t / r;
          v = (T)(0.5 * (xr * (double)h[off] + (1.0 + tr) * (double)h[i] - tr * xr * d));
        }
      }
    }
    out[i] = v;
  }
}

// Gamma_ij of the PSD Jacobian from the eigenvalues: 1 when both are > 0, 0 when both are <= 0, else
// lam_+ / (lam_+ - lam_-) (the branch forms, free of the cancellation of the difference quotient)
template <typename T>
__device__ __forceinline__ T sa_gamma(T li, T lj) {
  const bool pi = li > T(0), pj = lj > T(0);
  if (pi == pj) return pi ? T(1) : T(0);
  return pi ? li / (li - lj) : lj / (lj - li);
}

// Entry (i, j) of H = mat(h) of a real PSD cone: the svec triangle unscaled by sqrt 2 off the diagonal, a square cone
// symmetrised as project! does
template <typename T>
__device__ __forceinline__ T sa_psd_entry(const PsdConeDesc& d, const T* __restrict__ h, int i, int j) {
  const int N = d.N;
  const T* x = h + d.off;
  if (d.triangle) {
    const int a = i < j ? i : j, b = i < j ? j : i;
    const T v = x[svec_pos(a, b)];
    return a != b ? v * T(0.70710678118654752440) : v;
  }
  return (x[(long long)j * N + i] + x[(long long)i * N + j]) / T(2);
}

// out[cone] from the symmetric part of the N x N matrix S (leading dimension ld): the svec triangle (sqrt 2 off the
// diagonal) or the full square, symmetrised again as the square projection writes it
template <typename T>
__device__ __forceinline__ void sa_psd_store(const PsdConeDesc& d, const T* S, long long ld, T* __restrict__ out, long long e,
                                             long long stride) {
  const int N = d.N;
  if (d.triangle) {
    const long long tri = (long long)N * (N + 1) / 2;
    for (; e < tri; e += stride) {
      int j = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
      while ((long long)(j + 1) * (j + 2) / 2 <= e) ++j;
      while ((long long)j * (j + 1) / 2 > e) --j;
      const int i = (int)(e - (long long)j * (j + 1) / 2);
      const T v = (S[i + j * ld] + S[j + i * ld]) / T(2);
      out[d.off + e] = i == j ? v : T(1.41421356237309504880) * v;
    }
  } else {
    for (; e < (long long)N * N; e += stride) {
      const int i = (int)(e % N), j = (int)(e / N);
      out[d.off + e] = (S[i + j * ld] + S[j + i * ld]) / T(2);
    }
  }
}

// Dpi h on the small PSD cones, one CTA per cone in shared memory: H = mat(h), C = Gamma o (Q' H Q), out = svec(Q C Q').
// Q (column-major N x N) and lam of cone k start at q_off[k] and lam_off[k].  Two N x N buffers: S1, S2.
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_psd_small_apply_kernel(const PsdConeDesc* __restrict__ descs,
                                                                    const long long* __restrict__ q_off,
                                                                    const int* __restrict__ lam_off, const T* __restrict__ Qall,
                                                                    const T* __restrict__ lam_all, const T* __restrict__ h,
                                                                    T* __restrict__ out) {
  extern __shared__ unsigned char smem_raw[];
  const PsdConeDesc d = descs[blockIdx.x];
  const int N = d.N;
  const T* lam = lam_all + lam_off[blockIdx.x];
  if (N == 1) {
    if (threadIdx.x == 0) out[d.off] = lam[0] > T(0) ? h[d.off] : T(0);
    return;
  }
  const T* Q = Qall + q_off[blockIdx.x];
  const int ld = N | 1;
  T* S1 = reinterpret_cast<T*>(smem_raw);
  T* S2 = S1 + (size_t)ld * N;
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {
    const int i = e % N, j = e / N;
    S1[i + j * ld] = sa_psd_entry(d, h, i, j);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {   // S2 = H Q
    const int i = e % N, j = e / N;
    T acc = 0;
    for (int k = 0; k < N; ++k) acc += S1[i + k * ld] * Q[k + (long long)j * N];
    S2[i + j * ld] = acc;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {   // S1 = Gamma o (Q' S2)
    const int i = e % N, j = e / N;
    T acc = 0;
    for (int k = 0; k < N; ++k) acc += Q[k + (long long)i * N] * S2[k + j * ld];
    S1[i + j * ld] = sa_gamma(lam[i], lam[j]) * acc;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {   // S2 = Q S1
    const int i = e % N, j = e / N;
    T acc = 0;
    for (int k = 0; k < N; ++k) acc += Q[i + (long long)k * N] * S1[k + j * ld];
    S2[i + j * ld] = acc;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) {   // S1 = S2 Q'
    const int i = e % N, j = e / N;
    T acc = 0;
    for (int k = 0; k < N; ++k) acc += S2[i + k * ld] * Q[j + (long long)k * N];
    S1[i + j * ld] = acc;
  }
  __syncthreads();
  sa_psd_store(d, S1, ld, out, threadIdx.x, blockDim.x);
}

// large cones: H = mat(h) (N x N, column-major)
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_psd_load_kernel(PsdConeDesc d, const T* __restrict__ h, T* __restrict__ H) {
  const int N = d.N;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < (long long)N * N; e += (long long)gridDim.x * blockDim.x)
    H[e] = sa_psd_entry(d, h, (int)(e % N), (int)(e / N));
}

// large cones: C *= Gamma (Hadamard) and Qt = Q' for the second sandwich of bj_gemm_kernel products
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_psd_hadamard_kernel(int N, const T* __restrict__ lam, const T* __restrict__ Q,
                                                                 T* __restrict__ C, T* __restrict__ Qt) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < (long long)N * N; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % N), j = (int)(e / N);
    C[e] *= sa_gamma(lam[i], lam[j]);
    Qt[e] = Q[j + (long long)i * N];
  }
}

// large cones: out[cone] from S = Q C Q'
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_psd_store_kernel(PsdConeDesc d, const T* __restrict__ S, T* __restrict__ out) {
  sa_psd_store(d, S, d.N, out, blockIdx.x * (long long)blockDim.x + threadIdx.x, (long long)gridDim.x * blockDim.x);
}

// large cones after the block-Jacobi eigensolver: lam = diag(A) 2^pe, and the cone counted near a kink when an
// eigenvalue is within the band of max |w_s| of the cone (psd_cone_max_kernel)
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_psd_large_eig_kernel(int N, const T* __restrict__ A, const double* __restrict__ up,
                                                                  const unsigned long long* __restrict__ mx_bits,
                                                                  T* __restrict__ lam, int* __restrict__ counts) {
  const double f = *up;
  const double band = sa_kink_band<T>(__longlong_as_double((long long)*mx_bits));
  bool kink = false;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const T l = (T)((double)A[i + (long long)i * N] * f);
    lam[i] = l;
    kink = kink || fabs((double)l) <= band;
  }
  if (__syncthreads_or(kink) && threadIdx.x == 0) atomicAdd(counts + SA_CNT_PSD, 1);
}

// ---- the operator (I - M') lam ------------------------------------------------------------------------------------
// ls = [lam_x; -lam_s / rho], t0 = rho .* ls_s = -lam_s (the reduced CG right-hand side reads it)
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_op_rhs_kernel(int n, int m, const T* __restrict__ lam, const T* __restrict__ rho,
                                                           T* __restrict__ ls, T* __restrict__ t0) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x) {
    if (k < n) {
      ls[k] = lam[k];
    } else {
      const long long r = k - n;
      ls[k] = -lam[k] / rho[r];
      t0[r] = -lam[k];
    }
  }
}

// h = lam_s - 2 b
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_op_mid_kernel(int m, const T* __restrict__ lam_s, const T* __restrict__ b, T* __restrict__ h) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) h[r] = lam_s[r] - T(2) * b[r];
}

// out = lam - [sigma a; b + Dpi(lam_s - 2 b)]
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_op_out_kernel(int n, int m, const T* __restrict__ lam, const T* __restrict__ a,
                                                           const T* __restrict__ b, const T* __restrict__ dh, T sigma,
                                                           T* __restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x)
    out[k] = k < n ? lam[k] - sigma * a[k] : lam[k] - b[k - n] - dh[k - n];
}

// the right-hand side, first part: gw_x = D g_x, and h = gs~ + rho gy~ (gs~ = g_s / E, gy~ = E g_y / c) for Dpi
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_gw_kernel(int n, int m, const double* __restrict__ gx, const double* __restrict__ gy,
                                                       const double* __restrict__ gs, const T* __restrict__ D,
                                                       const T* __restrict__ E, double c, const T* __restrict__ rho,
                                                       T* __restrict__ gw, T* __restrict__ h) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x) {
    if (k < n) {
      gw[k] = gx ? (T)(D ? (double)D[k] * gx[k] : gx[k]) : T(0);
    } else {
      const long long r = k - n;
      const double e = E ? (double)E[r] : 1.0;
      const double gst = gs ? gs[r] / e : 0.0, gyt = gy ? e * gy[r] / c : 0.0;
      h[r] = (T)(gst + (double)rho[r] * gyt);
    }
  }
}

// the right-hand side, second part: gw_s = Dpi(gs~ + rho gy~) - rho gy~
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_gw_s_kernel(int m, const double* __restrict__ gy, const T* __restrict__ E, double c,
                                                         const T* __restrict__ rho, const T* __restrict__ dh, T* __restrict__ gw_s) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const double gyt = gy ? (E ? (double)E[r] : 1.0) * gy[r] / c : 0.0;
    gw_s[r] = (T)((double)dh[r] - (double)rho[r] * gyt);
  }
}

// ---- GMRES vector work --------------------------------------------------------------------------------------------
// part[c * gridDim.x + blockIdx.x] = block partial of V_c'w, c = blockIdx.y (V_c at V + c ldv), fp64 accumulation
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_dots_kernel(long long len, const T* __restrict__ V, long long ldv,
                                                         const T* __restrict__ w, double* __restrict__ part) {
  __shared__ double sm[kWarpsPerBlock];
  const T* v = V + blockIdx.y * ldv;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x)
    acc += (double)v[i] * (double)w[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = sm[0];
    for (int k = 1; k < kWarpsPerBlock; ++k) s += sm[k];
    part[blockIdx.y * gridDim.x + blockIdx.x] = s;
  }
}

// out[c] = sum of the nb partials of column c, in block order
__global__ void sa_fold_kernel(int k, int nb, const double* __restrict__ part, double* __restrict__ out) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < k; c += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nb; ++b) s += part[(long long)c * nb + b];
    out[c] = s;
  }
}

// w += alpha sum_c coef[c] V_c, the columns summed in order in fp64
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_axpy_kernel(long long len, const T* __restrict__ V, long long ldv, int k,
                                                         const double* __restrict__ coef, double alpha, T* __restrict__ w) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int c = 0; c < k; ++c) s += coef[c] * (double)V[c * ldv + i];
    w[i] = (T)((double)w[i] + alpha * s);
  }
}

// w /= sqrt(*nrm2) (0 stays 0: a breakdown)
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_normalise_kernel(long long len, const double* __restrict__ nrm2, T* __restrict__ w) {
  const double nv = sqrt(*nrm2);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x)
    w[i] = nv > 0.0 ? (T)((double)w[i] / nv) : T(0);
}

// r = g - r
template <typename T>
__global__ void __launch_bounds__(kBlock) sa_residual_kernel(long long len, const T* __restrict__ g, T* __restrict__ r) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x)
    r[i] = g[i] - r[i];
}

// ---- gradients ----------------------------------------------------------------------------------------------------
template <typename T>
struct SolveAdjointVecArgs {
  int n, m;
  const unsigned char* row_class;
  const unsigned char* flag;        // SA_ROW_* of the Nonnegatives and Box rows
  const T* box_l;
  const T* box_u;
  const T* u;                       // [u; v] = K^-1 [lam_x; -lam_s / rho]
  const T* v;
  const T* lam_s;
  const T* rho;
  const double* gy;                 // incoming gradients (null: zero)
  const double* gs;
  const T* D;                       // null: unscaled engine
  const T* E;
  double c;
  double* dq;                       // outputs, each may be null
  double* db;
  double* dl;
  double* du;
};

// dq = -c D u,  db = E v,  and on Box rows clamped at a bound  val = E (lam_s - 2 v + gs~ + rho gy~)  into dl (w_s <= l)
// or du (w_s >= u), half into each when l = u; 0 on every other row.  One thread per entry of [x; s].
template <typename T>
__global__ void __launch_bounds__(kBlock) solve_adjoint_grad_vec_kernel(SolveAdjointVecArgs<T> a) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)a.n + a.m; k += (long long)gridDim.x * blockDim.x) {
    if (k < a.n) {
      if (a.dq) a.dq[k] = -(a.D ? a.c * (double)a.D[k] : a.c) * (double)a.u[k];
      continue;
    }
    const int r = (int)(k - a.n);
    const double e = a.E ? (double)a.E[r] : 1.0;
    const double v = (double)a.v[r];
    if (a.db) a.db[r] = e * v;
    double lo = 0.0, up = 0.0;
    const unsigned char f = a.flag[r];
    if (a.row_class[r] == ROW_BOX && (f == SA_ROW_LOWER || f == SA_ROW_UPPER)) {
      const double gst = a.gs ? a.gs[r] / e : 0.0, gyt = a.gy ? e * a.gy[r] / a.c : 0.0;
      const double val = e * ((double)a.lam_s[r] - 2.0 * v + gst + (double)a.rho[r] * gyt);
      if (a.box_l[r] == a.box_u[r]) lo = up = 0.5 * val;
      else if (f == SA_ROW_LOWER) lo = val;
      else up = val;
    }
    if (a.dl) a.dl[r] = lo;
    if (a.du) a.du[r] = up;
  }
}

// ---- the forward derivative (cosmo_b200_solve_derivative, DESIGN.md §3l) -----------------------------------------
// The transpose of the operator above: for a data direction (dP, dq, dA, db, dl, du), scaled as the data are,
//   t = [x'; dPi - nu' / rho],  [x'; nu'] = K^-1 [-dq - dP x - dA' y; db - 2 dPi - dA x],  (I - M) w' = t  (GMRES),
//   (I - M) v = [v_x - a; v_s + b / rho - h],  h = Dpi v_s,  [a; b] = K^-1 [sigma v_x; v_s - 2 h],
//   x' = w'_x,  s' = Dpi w'_s + dPi,  y' = -rho (w'_s - s'),
// with dPi the Box term of the bound directions.  The direction passes below each write every output once, summing
// a warp's lanes through the fixed xor tree.

// map[p] = k for the CSR(A) position p of the CSC entry k, one warp per column j of A (row j of A', whose value order
// is A's CSC order): the row r of the entry, then j found by binary search among the ascending columns of CSR(A) row r
__global__ void __launch_bounds__(kBlock) sd_amap_kernel(int n, const int* __restrict__ at_rowptr, const int* __restrict__ at_col,
                                                         const int* __restrict__ a_rowptr, const int* __restrict__ a_col,
                                                         int* __restrict__ map) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += warps) {
    for (int k = at_rowptr[j] + lane; k < at_rowptr[j + 1]; k += 32) {
      const int r = at_col[k];
      int lo = a_rowptr[r], hi = a_rowptr[r + 1] - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a_col[mid] < j) lo = mid + 1;
        else hi = mid;
      }
      map[lo] = k;
    }
  }
}

// dPi of the Box rows from the scaled bound directions E dl, E du: dl~ where w_s <= l, du~ where w_s >= u, their mean
// on clamped rows with l = u, 0 on every other row (the transpose of solve_adjoint_grad_vec_kernel's split)
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_box_kernel(int m, const unsigned char* __restrict__ row_class,
                                                        const unsigned char* __restrict__ flag, const T* __restrict__ box_l,
                                                        const T* __restrict__ box_u, const double* __restrict__ dl,
                                                        const double* __restrict__ du, const T* __restrict__ E,
                                                        T* __restrict__ dpi) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    double v = 0.0;
    const unsigned char f = flag[r];
    if (row_class[r] == ROW_BOX && (f == SA_ROW_LOWER || f == SA_ROW_UPPER)) {
      const double e = E ? (double)E[r] : 1.0;
      const double lo = dl ? e * dl[r] : 0.0, up = du ? e * du[r] : 0.0;
      if (box_l[r] == box_u[r]) v = 0.5 * (lo + up);
      else v = f == SA_ROW_LOWER ? lo : up;
    }
    dpi[r] = (T)v;
  }
}

// ls_x = -c D_i dq_i - (dP~ x~)_i - (dA~' y~)_i, one warp per i over CSR(P) row i and CSR(A') row i (y = -mu):
//   dP~_ij = c D_i D_j dPx[src[k]],  dA~'_ir = E_r D_i dAx[k]  (A''s value order is A's CSC order)
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_rhs_x_kernel(int n, const int* __restrict__ p_rowptr, const int* __restrict__ p_col,
                                                          const int* __restrict__ p_src, const int* __restrict__ at_rowptr,
                                                          const int* __restrict__ at_col, const double* __restrict__ dPx,
                                                          const double* __restrict__ dq, const double* __restrict__ dAx,
                                                          const T* __restrict__ x, const T* __restrict__ mu,
                                                          const T* __restrict__ D, const T* __restrict__ E, double c,
                                                          T* __restrict__ ls) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    double px = 0.0, ay = 0.0;
    if (dPx)
      for (int k = p_rowptr[i] + lane; k < p_rowptr[i + 1]; k += 32) {
        const int j = p_col[k];
        px += (D ? (double)D[j] : 1.0) * dPx[p_src[k]] * (double)x[j];
      }
    if (dAx)
      for (int k = at_rowptr[i] + lane; k < at_rowptr[i + 1]; k += 32) {
        const int r = at_col[k];
        ay -= (E ? (double)E[r] : 1.0) * dAx[k] * (double)mu[r];
      }
    px = warp_sum(px);
    ay = warp_sum(ay);
    if (lane == 0) {
      const double di = D ? (double)D[i] : 1.0;
      ls[i] = (T)(-di * ((dq ? c * dq[i] : 0.0) + c * px + ay));
    }
  }
}

// ls_s = E_r db_r - 2 dPi_r - (dA~ x~)_r, one warp per CSR(A) row r (map: CSR position -> CSC index), t0 = rho .* ls_s
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_rhs_s_kernel(int m, const int* __restrict__ a_rowptr, const int* __restrict__ a_col,
                                                          const int* __restrict__ map, const double* __restrict__ dAx,
                                                          const double* __restrict__ db, const T* __restrict__ dpi,
                                                          const T* __restrict__ x, const T* __restrict__ D,
                                                          const T* __restrict__ E, const T* __restrict__ rho,
                                                          T* __restrict__ ls_s, T* __restrict__ t0) {
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
      const T v = (T)((db ? e * db[r] : 0.0) - 2.0 * (double)dpi[r] - acc);
      ls_s[r] = v;
      t0[r] = rho[r] * v;
    }
  }
}

// t = [x'; dPi - nu' / rho] from [x'; nu'] = K^-1 [ls_x; ls_s]
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_t_kernel(int n, int m, const T* __restrict__ xsol, const T* __restrict__ nu,
                                                      const T* __restrict__ dpi, const T* __restrict__ rho, T* __restrict__ t) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x)
    t[k] = k < n ? xsol[k] : dpi[k - n] - nu[k - n] / rho[k - n];
}

// ls = [sigma v_x; v_s - 2 h], t0 = rho .* ls_s (h = Dpi v_s)
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_op_rhs_kernel(int n, int m, const T* __restrict__ v, const T* __restrict__ h, T sigma,
                                                           const T* __restrict__ rho, T* __restrict__ ls, T* __restrict__ t0) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x) {
    if (k < n) {
      ls[k] = sigma * v[k];
    } else {
      const long long r = k - n;
      const T w = v[k] - T(2) * h[r];
      ls[k] = w;
      t0[r] = rho[r] * w;
    }
  }
}

// out = (I - M) v = [v_x - a; v_s + b / rho - h]
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_op_out_kernel(int n, int m, const T* __restrict__ v, const T* __restrict__ a,
                                                           const T* __restrict__ b, const T* __restrict__ h,
                                                           const T* __restrict__ rho, T* __restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x) {
    if (k < n) {
      out[k] = v[k] - a[k];
    } else {
      const long long r = k - n;
      out[k] = v[k] + b[r] / rho[r] - h[r];
    }
  }
}

// the outputs, unscaled: dx = D w'_x,  ds = s~' / E,  dy = -E rho (w'_s - s~') / c  with s~' = Dpi w'_s + dPi
template <typename T>
__global__ void __launch_bounds__(kBlock) sd_out_kernel(int n, int m, const T* __restrict__ w, const T* __restrict__ dh,
                                                        const T* __restrict__ dpi, const T* __restrict__ rho,
                                                        const T* __restrict__ D, const T* __restrict__ E, double c,
                                                        double* __restrict__ dx, double* __restrict__ dy, double* __restrict__ ds) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < (long long)n + m; k += (long long)gridDim.x * blockDim.x) {
    if (k < n) {
      if (dx) dx[k] = (D ? (double)D[k] : 1.0) * (double)w[k];
      continue;
    }
    const long long r = k - n;
    const double e = E ? (double)E[r] : 1.0;
    const double st = (double)dh[r] + (double)dpi[r];
    if (ds) ds[r] = st / e;
    if (dy) dy[r] = -e * (double)rho[r] * ((double)w[k] - st) / c;
  }
}

}  // namespace cosmo
