// ruiz.cuh -- Ruiz equilibration of the KKT data on the device (scale_ruiz!, scaling.jl:21-116).
//
// The reference rescales P, A, q, b in place `settings.scaling` times.  Here the matrices stay untouched while the
// scalings are being computed: with the running D, E, c the scaled data are
//     P_k = c D P0 D,   A_k = E A0 D,   q_k = c D q0,   b_k = E b0,
// so the column / row infinity norms the loop needs are weighted row maxima of the RESIDENT CSR copies
// (kkt_col_norms!, scaling.jl:3-8: columns of P and A = rows of P (symmetric) and of the stored A'; rows of A),
// and the final D, E, c are applied once to the CSR copies of A, A', P and to q, b, Box bounds; the column-windowed
// slabs are filled from the scaled A' afterwards (write_values in engine.cu).  No scalar ever visits the host inside
// the loop.
// Included from engine.cu (after spmv.cuh: CsrView).
#pragma once

namespace cosmo {

// out[r] = (acc ? max(out[r], v) : v),  v = scal * wrow[r] * max_k |val[k]| wcol[col[k]]     (one warp per row)
template <typename T>
__global__ void __launch_bounds__(kBlock) ruiz_row_inf_kernel(int nrows, CsrView<T> M, const T* __restrict__ wrow,
                                                              const T* __restrict__ wcol, const T* __restrict__ scal,
                                                              T* __restrict__ out, int acc) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nrows; r += warps) {
    const int s = M.rowptr[r], e = M.rowptr[r + 1];
    T mx = T(0);
    for (int k = s + lane; k < e; k += 32) mx = fmax(mx, fabs(M.val[k]) * wcol[M.col[k]]);
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) {
      T v = wrow[r] * mx;
      if (scal) v *= *scal;
      out[r] = acc ? fmax(out[r], v) : v;
    }
  }
}

// limit_scaling! + inv_sqrt! + lmul! (scaling.jl:10-13,62-71,125-127): work = 1 / sqrt(clip(work, lo, hi, 1, hi)); acc *= work
template <typename T>
__global__ void __launch_bounds__(kBlock) ruiz_update_kernel(int len, T* __restrict__ work, T* __restrict__ acc, T lo, T hi) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < len; i += gridDim.x * blockDim.x) {
    T w = work[i];
    w = (w < lo) ? T(1) : ((w > hi) ? hi : w);
    w = T(1) / sqrt(w);
    work[i] = w;
    acc[i] *= w;
  }
}

// cost scaling (scaling.jl:73-90), one block: mean of the column norms of the scaled P, |q|_inf of the scaled q, then
// c *= 1 / limit(max(limit(|q|_inf), mean))  when both are non-zero.  colnorm already contains the factor c.
template <typename T>
__global__ void __launch_bounds__(1024) ruiz_cost_kernel(int n, const T* __restrict__ colnorm, const T* __restrict__ q0,
                                                         const T* __restrict__ D, T* __restrict__ c, T lo, T hi) {
  __shared__ double ssum[32];
  __shared__ double smax[32];
  double sum = 0.0, mx = 0.0;
  const double cc = (double)*c;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    sum += (double)colnorm[i];
    mx = fmax(mx, fabs(cc * (double)D[i] * (double)q0[i]));
  }
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { ssum[threadIdx.x >> 5] = sum; smax[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0, m = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { s += ssum[w]; m = fmax(m, smax[w]); }
    const double mean = n ? s / (double)n : 0.0;
    if (mean != 0.0 && m != 0.0) {
      auto lim = [&](double v) { return (v < (double)lo) ? 1.0 : ((v > (double)hi) ? (double)hi : v); };
      const double qn = lim(m);
      const double sc = lim(qn > mean ? qn : mean);
      *c = (T)(cc * (1.0 / sc));
    }
  }
}

// rectify_scaling! for cones that admit only a scalar scaling (convexset.jl:905-958): Ew = mean(E[cone]) ./ E[cone];
// E .*= Ew.  One block per cone.
template <typename T>
__global__ void __launch_bounds__(kBlock) ruiz_rectify_kernel(const int* __restrict__ cone_off, const int* __restrict__ cone_dim,
                                                              T* __restrict__ E) {
  __shared__ double red[kWarpsPerBlock];
  __shared__ double mean_s;
  const int off = cone_off[blockIdx.x], dim = cone_dim[blockIdx.x];
  double s = 0.0;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) s += (double)E[off + i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kWarpsPerBlock; ++w) t += red[w];
    mean_s = t / (double)dim;
  }
  __syncthreads();
  const T mean = (T)mean_s;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) {
    const T e = E[off + i];
    E[off + i] = e * (mean / e);
  }
}

// val[k] *= scal * (wrow[r] * wcol[col[k]])   (plain CSR copy)
// The product wrow[r] * wcol[col[k]] is taken first: for P (both triangles stored, wrow = wcol = D) it is D_i D_j on
// both sides of the diagonal, bit for bit, so the scaled P is exactly symmetric, as the reference makes it with
// symmetrize_full! (scaling.jl:99).  Scaling (scal * D_i) first would round P_ij and P_ji differently.  Without scal the
// factor is exactly 1 and A, A' get E_i D_j.
template <typename T>
__global__ void __launch_bounds__(kBlock) ruiz_apply_csr_kernel(int nrows, const int* __restrict__ rowptr, const int* __restrict__ col,
                                                                T* __restrict__ val, const T* __restrict__ wrow,
                                                                const T* __restrict__ wcol, const T* __restrict__ scal) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const T sc = scal ? *scal : T(1);
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nrows; r += warps) {
    const int s = rowptr[r], e = rowptr[r + 1];
    const T wr = wrow[r];
    for (int k = s + lane; k < e; k += 32) val[k] *= sc * (wr * wcol[col[k]]);
  }
}

// q = c D q0;  Dinv = 1 / D
template <typename T>
__global__ void __launch_bounds__(kBlock) ruiz_finish_n_kernel(int n, T* __restrict__ q, const T* __restrict__ D, T* __restrict__ Dinv,
                                                               const T* __restrict__ c) {
  const T cc = *c;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    q[i] = cc * D[i] * q[i];
    Dinv[i] = T(1) / D[i];
  }
}

// b = E b0;  Einv = 1 / E;  Box bounds: l .*= E, u .*= E (scale!(::Box), convexset.jl:863-867)
template <typename T>
__global__ void __launch_bounds__(kBlock) ruiz_finish_m_kernel(int m, T* __restrict__ b, const T* __restrict__ E, T* __restrict__ Einv,
                                                               const unsigned char* __restrict__ row_class, T* __restrict__ box_l,
                                                               T* __restrict__ box_u) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const T e = E[i];
    b[i] = e * b[i];
    Einv[i] = T(1) / e;
    if (row_class[i] == ROW_BOX) { box_l[i] *= e; box_u[i] *= e; }
  }
}

template <typename T>
__global__ void ruiz_fill_kernel(int len, T* __restrict__ v, T x) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < len; i += gridDim.x * blockDim.x) v[i] = x;
}

}  // namespace cosmo
