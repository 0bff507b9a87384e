// vector_kernels.cuh -- fused elementwise / reduction kernels of the ADMM loop
// (K4, K5, K7-K9, K12 of SURVEY.md 2a).  All HBM-bound, grid-stride, 256 threads.
#pragma once
#include "common.cuh"

namespace cosmo {

// device-resident scalars of the inner Krylov solvers (indices into T* sc / int* isc)
enum {
  SC_RES = 0,    // |r|_2
  SC_PREV = 1,   // previous |r|_2
  SC_TOL = 2,    // absolute tolerance
  SC_RES2 = 3,   // reduction slot: |r|^2
  SC_RHS2 = 4,   // reduction slot: |rhs|^2 (must follow SC_RES2)
  SC_TMP0 = 5,   // scratch reduction slots
  SC_TMP1 = 6,
  SC_TMP2 = 7,
  SC_TMP3 = 8,
  SC_TMP4 = 9,
  SC_TMP5 = 10,
  SC_TMP6 = 11,
  SC_TMP7 = 12,
  // MINRES state (IterativeSolvers minres.jl)
  SC_H1 = 16, SC_H2 = 17, SC_H3 = 18, SC_H4 = 19,
  SC_RHS_1 = 20, SC_RHS_2 = 21,
  SC_C_PREV = 22, SC_S_PREV = 23, SC_C_CURR = 24, SC_S_CURR = 25,
  // per-iteration coefficients handed from the scalar epilogue to the vector update kernel
  SC_K3_INV_H4 = 26, SC_K3_H2 = 27, SC_K3_H1 = 28, SC_K3_INV_H3 = 29, SC_K3_RHS1 = 30,
  SC_COUNT = 32
};
enum { ISC_DONE = 0, ISC_IT = 1, ISC_MAXIT = 2, ISC_COUNT = 8 };

// cone classes per row
enum : unsigned char { ROW_ZERO = 0, ROW_NONNEG = 1, ROW_BOX = 2, ROW_SOC = 3, ROW_PSD = 4, ROW_CONE3 = 5, ROW_CUSTOM = 6 };

template <typename T>
struct SocTable {          // one entry per SecondOrderCone
  const int* off;          // first row of the cone
  const T* norm;           // |x[2:end]|_2 of the current w_s (written by soc kernels)
};

// ---------------------------------------------------------------------------
// K5 + K7: s = Pi_K(w_s) for the elementwise cones and the SOC scaling, fused
// with the right-hand side of the x-step (solver.jl:14-15, 50-51; convexset.jl
// :25-28, 71-74, 100-114, 844-847; kktsolver_indirect.jl:52):
//   ls_x = sigma w_x - q ;  x2 = b - 2 s + w_s ;  t0 = rho .* x2
// PSD rows are written by the PSD kernels beforehand (s already holds them).
// ---------------------------------------------------------------------------
template <typename T>
struct ProjRhsArgs {
  int n, m;
  const T* w;        // operator variable [w_x; w_s] the projection reads
  const T* ws_rhs;   // w_s used to build the rhs (differs from w+n after a rho update, solver.jl:278)
  const T* q;
  const T* b;
  const T* rho;
  const T* box_l;    // m-length, only read on BOX rows
  const T* box_u;
  const unsigned char* row_class;
  const int* row_cone;   // SOC rows: index into the SOC table
  SocTable<T> soc;
  T* s;
  T* ls;             // [x1; x2]
  T* t0;             // rho .* x2
  T sigma;
  int do_proj, do_rhs;
};

template <typename T>
__global__ void __launch_bounds__(kBlock) proj_rhs_kernel(ProjRhsArgs<T> a) {
  const int total = a.n + a.m;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    if (idx < a.n) {
      if (a.do_rhs) a.ls[idx] = a.sigma * a.w[idx] - a.q[idx];
      continue;
    }
    const int r = idx - a.n;
    T sv;
    if (a.do_proj) {
      const T ws = a.w[a.n + r];
      const unsigned char cls = a.row_class[r];
      if (cls == ROW_ZERO) {
        sv = T(0);
      } else if (cls == ROW_NONNEG) {
        sv = (ws > T(0)) ? ws : ((ws != ws) ? ws : T(0));
      } else if (cls == ROW_BOX) {
        const T l = a.box_l[r], u = a.box_u[r];
        sv = (ws < l) ? l : ((ws > u) ? u : ws);   // clip, algebra.jl:5-7
      } else if (cls == ROW_SOC) {
        const int k = a.row_cone[r];
        const int off = a.soc.off[k];
        const T t = a.w[a.n + off];
        const T nx = a.soc.norm[k];
        if (nx <= t) sv = ws;
        else if (nx <= -t) sv = T(0);
        else sv = (r == off) ? (nx + t) / T(2) : (nx + t) / (T(2) * nx) * ws;
      } else {
        sv = a.s[r];   // PSD, Exp/Pow and custom rows: projected by their own kernels beforehand
      }
      a.s[r] = sv;
    } else {
      sv = a.s[r];
    }
    if (a.do_rhs) {
      const T x2 = a.b[r] - T(2) * sv + a.ws_rhs[r];
      a.ls[idx] = x2;
      a.t0[r] = a.rho[r] * x2;
    }
  }
}

// The same pass with 128-bit loads and stores: one thread owns TWO consecutive entries of [w_x; w_s] (fp64; four for
// fp32 would need another unroll and is left to the scalar kernel).  Requires n even, so that the m-part of every
// (n+m)-vector starts 16-byte aligned like the m-vectors do; the host picks the scalar kernel otherwise.  The cone
// class is read as one 16-bit load per pair; SOC / PSD / Exp rows take the scalar formulas per element.
template <typename T>
__device__ __forceinline__ T proj_row_scalar(const ProjRhsArgs<T>& a, int r, T ws, unsigned char cls) {
  if (cls == ROW_ZERO) return T(0);
  if (cls == ROW_NONNEG) return (ws > T(0)) ? ws : ((ws != ws) ? ws : T(0));
  if (cls == ROW_BOX) {
    const T l = a.box_l[r], u = a.box_u[r];
    return (ws < l) ? l : ((ws > u) ? u : ws);
  }
  if (cls == ROW_SOC) {
    const int k = a.row_cone[r];
    const int off = a.soc.off[k];
    const T t = a.w[a.n + off];
    const T nx = a.soc.norm[k];
    if (nx <= t) return ws;
    if (nx <= -t) return T(0);
    return (r == off) ? (nx + t) / T(2) : (nx + t) / (T(2) * nx) * ws;
  }
  return a.s[r];   // PSD, Exp/Pow and custom rows: projected by their own kernels beforehand
}

__global__ void __launch_bounds__(kBlock) proj_rhs_vec2_kernel(ProjRhsArgs<double> a) {
  const int npx = a.n >> 1;                      // pairs in the x-part (n even)
  const int npairs = npx + ((a.m + 1) >> 1);
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += gridDim.x * blockDim.x) {
    if (p < npx) {
      if (a.do_rhs) {
        const double2 w = reinterpret_cast<const double2*>(a.w)[p];
        const double2 q = reinterpret_cast<const double2*>(a.q)[p];
        reinterpret_cast<double2*>(a.ls)[p] = make_double2(a.sigma * w.x - q.x, a.sigma * w.y - q.y);
      }
      continue;
    }
    const int r = (p - npx) << 1;
    if (r + 1 >= a.m) {                           // odd tail row
      double sv;
      if (a.do_proj) { sv = proj_row_scalar<double>(a, r, a.w[a.n + r], a.row_class[r]); a.s[r] = sv; }
      else sv = a.s[r];
      if (a.do_rhs) {
        const double x2 = a.b[r] - 2.0 * sv + a.ws_rhs[r];
        a.ls[a.n + r] = x2;
        a.t0[r] = a.rho[r] * x2;
      }
      continue;
    }
    double2 sv;
    if (a.do_proj) {
      const double2 ws = *reinterpret_cast<const double2*>(a.w + a.n + r);
      const unsigned short c2 = *reinterpret_cast<const unsigned short*>(a.row_class + r);
      const unsigned char c0 = (unsigned char)(c2 & 0xff), c1 = (unsigned char)(c2 >> 8);
      if (c0 == ROW_BOX && c1 == ROW_BOX) {       // the common long run: vector loads of the bounds
        const double2 l = *reinterpret_cast<const double2*>(a.box_l + r);
        const double2 u = *reinterpret_cast<const double2*>(a.box_u + r);
        sv.x = (ws.x < l.x) ? l.x : ((ws.x > u.x) ? u.x : ws.x);
        sv.y = (ws.y < l.y) ? l.y : ((ws.y > u.y) ? u.y : ws.y);
      } else {
        sv.x = proj_row_scalar<double>(a, r, ws.x, c0);
        sv.y = proj_row_scalar<double>(a, r + 1, ws.y, c1);
      }
      *reinterpret_cast<double2*>(a.s + r) = sv;
    } else {
      sv = *reinterpret_cast<const double2*>(a.s + r);
    }
    if (a.do_rhs) {
      const double2 b = *reinterpret_cast<const double2*>(a.b + r);
      const double2 wr = *reinterpret_cast<const double2*>(a.ws_rhs + r);
      const double2 rho = *reinterpret_cast<const double2*>(a.rho + r);
      const double2 x2 = make_double2(b.x - 2.0 * sv.x + wr.x, b.y - 2.0 * sv.y + wr.y);
      *reinterpret_cast<double2*>(a.ls + a.n + r) = x2;
      *reinterpret_cast<double2*>(a.t0 + r) = make_double2(rho.x * x2.x, rho.y * x2.y);
    }
  }
}

constexpr int kSocZeroExp = -100000;   // exponent recorded for an all-zero chunk (exact in float and double)

// SOC norms, stage 1: one block per chunk of a cone's tail (deterministic tree).  The squares are summed after scaling
// the chunk by the power of two 2^-e nearest its maximum (exact), so the sum neither overflows nor underflows anywhere in
// the range of T; chunk_sum[2 c] = the scaled sum, chunk_sum[2 c + 1] = e.
template <typename T>
__global__ void __launch_bounds__(kBlock) soc_chunk_kernel(const T* __restrict__ ws, const int* __restrict__ chunk_start,
                                                           const int* __restrict__ chunk_len, T* __restrict__ chunk_sum) {
  __shared__ T sm[kWarpsPerBlock];
  const int c = blockIdx.x;
  const int start = chunk_start[c], len = chunk_len[c];
  T mx = 0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) mx = fmax(mx, tabs(ws[start + i]));
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = sm[0];
  for (int w = 1; w < kWarpsPerBlock; ++w) mx = fmax(mx, sm[w]);
  __syncthreads();
  // an all-zero chunk contributes nothing and must not set the common exponent of the cone: kSocZeroExp keeps it out
  const int e = (mx == T(0)) ? kSocZeroExp : pow2_exponent(mx);
  const T inv = (mx == T(0)) ? T(1) : (T)ldexp(1.0, -e);
  T acc = 0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const T v = ws[start + i] * inv;
    acc += v * v;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    T v = sm[0];
    for (int w = 1; w < kWarpsPerBlock; ++w) v += sm[w];
    chunk_sum[2 * c] = v;
    chunk_sum[2 * c + 1] = (T)e;
  }
}

// SOC norms, stage 2: one thread per cone folds its chunks in order, relative to the largest chunk exponent E:
// norm = 2^E sqrt(sum_c s_c 4^(e_c - E)).
template <typename T>
__global__ void soc_final_kernel(const T* __restrict__ chunk_sum, const int* __restrict__ cone_chunk_ptr, int ncones,
                                 T* __restrict__ norm) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ncones) return;
  int E = kSocZeroExp;
  for (int c = cone_chunk_ptr[k]; c < cone_chunk_ptr[k + 1]; ++c) E = max(E, (int)chunk_sum[2 * c + 1]);
  T v = 0;
  for (int c = cone_chunk_ptr[k]; c < cone_chunk_ptr[k + 1]; ++c) {
    const int ec = (int)chunk_sum[2 * c + 1];
    if (ec != kSocZeroExp) v += chunk_sum[2 * c] * (T)ldexp(1.0, 2 * (ec - E));
  }
  norm[k] = (v == T(0)) ? T(0) : (T)ldexp((double)sqrt(v), E);
}

// w_x <- w_x + alpha (x_tl - w_x)              (solver.jl:63), ping-pong buffers
template <typename T>
__global__ void __launch_bounds__(kBlock) wx_update_kernel(int n, const T* __restrict__ w_in, const T* __restrict__ xtl,
                                                           T alpha, T* __restrict__ w_out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T w = w_in[i];
    w_out[i] = w + alpha * (xtl[i] - w);
  }
}

// mu = rho .* (w_prev_s - s)                    (recover_mu!, solver.jl:24-26)
template <typename T>
__global__ void __launch_bounds__(kBlock) recover_mu_kernel(int m, const T* __restrict__ rho, const T* __restrict__ wps,
                                                            const T* __restrict__ s, T* __restrict__ mu) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x)
    mu[i] = rho[i] * (wps[i] - s[i]);
}

// w_s = mu ./ rho + s                           (solver.jl:129, :278)
template <typename T>
__global__ void __launch_bounds__(kBlock) ws_from_mu_kernel(int m, const T* __restrict__ rho, const T* __restrict__ mu,
                                                            const T* __restrict__ s, T* __restrict__ ws) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x)
    ws[i] = T(1) / rho[i] * mu[i] + s[i];
}

// rho_class of every row (classify_constraints!, setup.jl:75-85; convexset.jl:62-69, 831-842), the table rho_vec_kernel
// reads: 1 on Zero rows and on Box rows with u - l < RHO_TOL, 2 on loose rows (Nonnegatives with b > big, Box with
// l < -big and u > big), 0 elsewhere.  Every comparison and u - l are taken in fp64 after widening the T values, so an
// fp32 engine classifies the numbers it holds exactly as an fp64 statement of the rule does; NaN compares false.
template <typename T>
__global__ void __launch_bounds__(kBlock) rho_class_kernel(int m, const unsigned char* __restrict__ row_class,
                                                           const T* __restrict__ b, const T* __restrict__ box_l,
                                                           const T* __restrict__ box_u, double big, double rho_tol,
                                                           unsigned char* __restrict__ rho_class) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const unsigned char cls = row_class[i];
    unsigned char c = 0;
    if (cls == ROW_ZERO) {
      c = 1;
    } else if (cls == ROW_NONNEG) {
      if ((double)b[i] > big) c = 2;
    } else if (cls == ROW_BOX) {
      const double l = (double)box_l[i], u = (double)box_u[i];
      if (l < -big && u > big) c = 2;
      else if (u - l < rho_tol) c = 1;
    }
    rho_class[i] = c;
  }
}

// rho_vec from the per-row class table        (parameters.jl:17-49, 75-81)
//   class 0: rho ; 1: rho * RHO_EQ_OVER_RHO_INEQ ; 2: RHO_MIN
template <typename T>
__global__ void __launch_bounds__(kBlock) rho_vec_kernel(int m, const unsigned char* __restrict__ rho_class, T rho,
                                                         T rho_eq_mult, T rho_min, T* __restrict__ rho_vec) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const unsigned char c = rho_class[i];
    rho_vec[i] = (c == 2) ? rho_min : ((c == 1) ? rho * rho_eq_mult : rho);
  }
}

template <typename T>
__global__ void __launch_bounds__(kBlock) scale_kernel(int n, const T* __restrict__ a, const T* x, T* y) {   // y may alias x
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = a[i] * x[i];
}

// y = a - b
template <typename T>
__global__ void __launch_bounds__(kBlock) sub_kernel(int n, const T* a, const T* __restrict__ b, T* y) {   // y may alias a
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = a[i] - b[i];
}

// ---------------------------------------------------------------------------
// CG on the reduced KKT system (IterativeSolvers.jl v0.9 cg!, called from
// kktsolver_indirect.jl:70).  Scalars live on the device; every kernel is a
// no-op once isc[ISC_DONE] is set so the host can enqueue iterations ahead.
// ---------------------------------------------------------------------------
// sum of the ranks' partial vectors at index i, in rank order (one-shot allreduce on the fly).  The partials were PUSHED
// into this rank's own buffer by p2p_push_kernel (segment slot * nranks + r holds rank r's vector): local reads only.
template <typename T>
__device__ __forceinline__ T p2p_gather(const P2pView<T>& v, unsigned slot, int i) {
  const T* base = v.peer_data[v.rank] + (size_t)slot * v.nranks * v.stride + i;
  T acc = ld_peer(base);
  for (int r = 1; r < v.nranks; ++r) acc += ld_peer(base + (size_t)r * v.stride);
  return acc;
}

// Producer side of the exchange: copy this rank's partial vector (len elements, len = n + 1 with the partial dot
// product riding at the end) into segment (slot, rank) of every peer's buffer over NVLink with coalesced 16-byte
// stores -- blockIdx.y = destination rank -- then publish the sequence number to that destination (last CTA of the
// destination, after a system-scope fence of every contributing CTA).
template <typename T>
__global__ void __launch_bounds__(kBlock) p2p_push_kernel(P2pView<T> v, const T* __restrict__ src, int len, const int* __restrict__ done,
                                                          unsigned* __restrict__ arrive) {
  if (done != nullptr && *done) return;
  const unsigned sq = *v.seq;
  const unsigned slot = sq & 1u;
  const int dst = blockIdx.y;
  T* out = v.peer_data[dst] + ((size_t)slot * v.nranks + v.rank) * v.stride;
  constexpr int VEC = 16 / (int)sizeof(T);
  const int nvec = len / VEC;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x)
    reinterpret_cast<int4*>(out)[i] = reinterpret_cast<const int4*>(src)[i];       // src and out are 16-byte aligned
  for (int i = nvec * VEC + blockIdx.x * blockDim.x + threadIdx.x; i < len; i += gridDim.x * blockDim.x) out[i] = src[i];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(arrive + dst, 1u);
    if (t == gridDim.x - 1) {
      arrive[dst] = 0;
      __threadfence_system();
      st_release_sys(v.peer_flags[dst] + slot * kMaxRanks + v.rank, sq + 1u);
    }
  }
}

template <typename T>
struct CgInitFin {
  T* sc; int* isc; T tol_num;
  unsigned* seq;   // non-null in peer-exchange mode: this consumer retires the sequence number
  __device__ void operator()(T* out) const {   // out[0] = |r|^2, out[1] = |rhs|^2
    const T res = sqrt(out[0]);
    const T rhsn = sqrt(out[1]);
    const T tol = tol_num / rhsn;              // abstol = get_tolerance(S)/norm(y1), reltol = 0
    sc[SC_RES] = res;
    sc[SC_PREV] = T(1);
    sc[SC_TOL] = tol;
    isc[ISC_IT] = 0;
    isc[ISC_DONE] = (res <= tol || isc[ISC_MAXIT] <= 0) ? 1 : 0;
    if (seq) *seq = *seq + 1u;
  }
};

// r = rhs - c (c = L x0) ; u = 0 ; |r|^2, |rhs|^2
template <typename T>
__global__ void __launch_bounds__(kBlock) cg_init_kernel(int n, const T* __restrict__ rhs, const T* __restrict__ c,
                                                         T* __restrict__ r, T* __restrict__ u, RedBuf<T> rb,
                                                         CgInitFin<T> fin, bool p2p, P2pView<T> xv) {
  pdl_launch_dependents();
  pdl_wait();
  T accS[2] = {0, 0};
  T accM[1] = {0};
  unsigned slot = 0;
  if (p2p) {
    const unsigned sq = *xv.seq;
    slot = sq & 1u;
    p2p_wait_all(xv, slot, sq + 1u);
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T b = rhs[i];
    const T ci = p2p ? p2p_gather(xv, slot, i) : c[i];
    const T ri = b - ci;
    r[i] = ri;
    u[i] = T(0);
    accS[0] += ri * ri;
    accS[1] += b * b;
  }
  reduce_and_finalize<T, 2, 0>(accS, accM, rb, fin);
}

// u = r + beta u,  beta = res^2 / prev^2
template <typename T>
__global__ void __launch_bounds__(kBlock) cg_update_u_kernel(int n, const T* __restrict__ r, T* __restrict__ u,
                                                             const T* __restrict__ sc, const int* __restrict__ isc) {
  pdl_launch_dependents();
  pdl_wait();
  if (isc[ISC_DONE]) return;
  const T res = sc[SC_RES], prev = sc[SC_PREV];
  const T beta = (res * res) / (prev * prev);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) u[i] = r[i] + beta * u[i];
}

template <typename T>
struct CgStepFin {
  T* sc; int* isc;
  unsigned* seq;
  __device__ void operator()(T* out) const {   // out[0] = |r|^2
    const T res = sqrt(out[0]);
    sc[SC_PREV] = sc[SC_RES];
    sc[SC_RES] = res;
    const int it = isc[ISC_IT] + 1;
    isc[ISC_IT] = it;
    isc[ISC_DONE] = (res <= sc[SC_TOL] || it >= isc[ISC_MAXIT]) ? 1 : 0;
    if (seq) *seq = *seq + 1u;
  }
};

// alpha = res^2 / (u'c) ; x += alpha u ; r -= alpha c ; |r|^2
template <typename T>
__global__ void __launch_bounds__(kBlock) cg_update_xr_kernel(int n, const T* __restrict__ u, const T* __restrict__ c,
                                                              const T* __restrict__ dot_uc, T* __restrict__ x,
                                                              T* __restrict__ r, const T* __restrict__ sc,
                                                              const int* __restrict__ isc, RedBuf<T> rb,
                                                              CgStepFin<T> fin, bool p2p, P2pView<T> xv) {
  pdl_launch_dependents();
  pdl_wait();
  if (isc[ISC_DONE]) return;
  const T res = sc[SC_RES];
  unsigned slot = 0;
  T dot;
  if (p2p) {
    const unsigned sq = *xv.seq;
    slot = sq & 1u;
    p2p_wait_all(xv, slot, sq + 1u);
    dot = p2p_gather(xv, slot, n);
  } else {
    dot = dot_uc[0];
  }
  const T alpha = (res * res) / dot;
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    x[i] += alpha * u[i];
    const T ci = p2p ? p2p_gather(xv, slot, i) : c[i];
    const T ri = r[i] - alpha * ci;
    r[i] = ri;
    accS[0] += ri * ri;
  }
  reduce_and_finalize<T, 1, 0>(accS, accM, rb, fin);
}

// ---------------------------------------------------------------------------
// generic reductions used by the infeasibility tests (infeasibility.jl, algebra.jl:9-47)
// ---------------------------------------------------------------------------
// out[0] = |scale .* v|_inf
template <typename T>
__global__ void __launch_bounds__(kBlock) scaled_norminf_kernel(int n, const T* __restrict__ scale,
                                                                const T* __restrict__ v, RedBuf<T> rb) {
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    accM[0] = nanmax(accM[0], tabs((scale ? scale[i] : T(1)) * v[i]));
  reduce_and_finalize<T, 0, 1>(accS, accM, rb, NoFin());
}

// out[0] = a'b
template <typename T>
__global__ void __launch_bounds__(kBlock) dot_kernel(int n, const T* __restrict__ a, const T* __restrict__ b,
                                                     RedBuf<T> rb) {
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) accS[0] += a[i] * b[i];
  reduce_and_finalize<T, 1, 0>(accS, accM, rb, NoFin());
}

// y = a * x (scalar a), elementwise
template <typename T>
__global__ void __launch_bounds__(kBlock) scal_kernel(int n, T a, T* __restrict__ x) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) x[i] *= a;
}

// Per-row certificates for the elementwise cones.
//   mode 0 (primal, infeasibility.jl:19-24 + convexset.jl:30-36,76-78,850-856):
//     v = -dy/|dy| rows;  sums[0] += Box support term (v>tol ? v*u : v*l),
//     max[0] = 1 if a NONNEG row violates in_dual(-v): (-v) < -tol  <=> v > tol
//   mode 1 (dual, infeasibility.jl:52-62 + convexset.jl:34-36,80-82,858-860):
//     v = Einv*A*dx/|dx| rows;  max[0] = 1 if any row leaves the polar recession cone
template <typename T>
__global__ void __launch_bounds__(kBlock) cone_rows_certificate_kernel(int m, int mode, const T* __restrict__ v,
                                                                      const unsigned char* __restrict__ row_class,
                                                                      const T* __restrict__ box_l,
                                                                      const T* __restrict__ box_u, T tol, RedBuf<T> rb) {
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const unsigned char cls = row_class[i];
    const T x = v[i];
    if (mode == 0) {
      if (cls == ROW_NONNEG) {
        if (x > tol) accM[0] = T(1);          // in_dual(-x): any(-x < -tol)
      } else if (cls == ROW_BOX) {
        accS[0] += (tabs(x) > tol && x > T(0)) ? x * box_u[i] : x * box_l[i];
      }
    } else {
      bool bad = false;
      if (cls == ROW_ZERO) bad = tabs(x) > tol;
      else if (cls == ROW_NONNEG) bad = x > tol;
      else if (cls == ROW_BOX) bad = (box_u[i] == INFINITY && x > tol) || (box_l[i] == -INFINITY && x < -tol);
      if (bad) accM[0] = T(1);
    }
  }
  reduce_and_finalize<T, 1, 1>(accS, accM, rb, NoFin());
}

// SOC certificate shared by both infeasibility tests (convexset.jl:116-122 via :919-923):
//   -v in K* (primal)  <=>  v in polar recession cone (dual)  <=>  |v[2:]|_2 <= tol - v[1]
// flag[0] = 1 if any cone violates it.  Single block.
template <typename T>
__global__ void __launch_bounds__(kBlock) soc_cert_kernel(int ncones, const int* __restrict__ off, const T* __restrict__ norm,
                                                          const T* __restrict__ v, T tol, T* __restrict__ flag) {
  int bad = 0;
  for (int k = threadIdx.x; k < ncones; k += blockDim.x)
    if (!(norm[k] <= tol - v[off[k]])) bad = 1;
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) flag[0] = bad ? T(1) : T(0);
}

// ---------------------------------------------------------------------------
// MINRES (IterativeSolvers.jl v0.9 minres!, called from kktsolver_indirect.jl:73,152)
// on an L-vector (L = n: reduced system, L = n+m: full KKT).  H[1..4], rhs[1..2] and
// the two stored Givens rotations live in sc[SC_H1..]; every kernel is a no-op once
// isc[ISC_DONE] is set, except the vector update of the iteration that set it.
// ---------------------------------------------------------------------------
template <typename T>
struct MinresInitFin {
  T* sc; int* isc; T tol_num;
  __device__ void operator()(T* out) const {   // out[0] = |b - L x|^2
    const T res = sqrt(out[0]);
    sc[SC_RES] = res;
    sc[SC_TOL] = tol_num / res;                // abstol = get_tolerance(S) / init_residual, reltol = 0
    sc[SC_H1] = sc[SC_H2] = sc[SC_H3] = sc[SC_H4] = T(0);
    sc[SC_RHS_1] = res; sc[SC_RHS_2] = T(0);
    sc[SC_C_PREV] = T(1); sc[SC_S_PREV] = T(0); sc[SC_C_CURR] = T(1); sc[SC_S_CURR] = T(0);
    isc[ISC_IT] = 0;
    isc[ISC_DONE] = (res <= sc[SC_TOL] || isc[ISC_MAXIT] <= 0) ? 1 : 0;
  }
};

// v_curr = b - c ; |v_curr|^2
template <typename T>
__global__ void __launch_bounds__(kBlock) minres_init_kernel(int L, const T* __restrict__ b, const T* __restrict__ c,
                                                             T* __restrict__ v_curr, RedBuf<T> rb, MinresInitFin<T> fin) {
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    const T v = b[i] - c[i];
    v_curr[i] = v;
    accS[0] += v * v;
  }
  reduce_and_finalize<T, 1, 0>(accS, accM, rb, fin);
}

// v_curr /= resnorm ; v_prev = w_prev = w_curr = 0
template <typename T>
__global__ void __launch_bounds__(kBlock) minres_start_kernel(int L, T* __restrict__ v_curr, T* __restrict__ v_prev,
                                                              T* __restrict__ w_prev, T* __restrict__ w_curr,
                                                              const T* __restrict__ sc) {
  const T inv = T(1) / sc[SC_RES];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    v_curr[i] *= inv;
    v_prev[i] = T(0);
    w_prev[i] = T(0);
    w_curr[i] = T(0);
  }
}

struct MinresProjFin {
  template <typename T>
  __device__ void operator()(T*) const {}
};

// v_next = c - H[2] v_prev ; proj = v_curr' v_next  -> sc[SC_H3]
template <typename T>
__global__ void __launch_bounds__(kBlock) minres_lanczos1_kernel(int L, const T* __restrict__ c, const T* __restrict__ v_prev,
                                                                 const T* __restrict__ v_curr, T* __restrict__ v_next,
                                                                 const T* __restrict__ sc, const int* __restrict__ isc,
                                                                 RedBuf<T> rb) {
  if (isc[ISC_DONE]) return;
  const T h2 = sc[SC_H2];
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    const T v = c[i] - h2 * v_prev[i];
    v_next[i] = v;
    accS[0] += v_curr[i] * v;
  }
  reduce_and_finalize<T, 1, 0>(accS, accM, rb, NoFin());
}

// LinearAlgebra.givensAlgorithm, real case: [c s; -s c] [f; g] = [r; 0]
template <typename T>
__device__ __forceinline__ void givens_rot(T f, T g, T& c, T& s, T& r) {
  if (g == T(0)) { c = T(1); s = T(0); r = f; return; }
  if (f == T(0)) { c = T(0); s = T(1); r = g; return; }
  r = hypot(f, g);
  c = f / r;
  s = g / r;
  if (tabs(f) > tabs(g) && c < T(0)) { c = -c; s = -s; r = -r; }
}

template <typename T>
struct MinresStepFin {
  T* sc; int* isc;
  __device__ void operator()(T* out) const {   // out[0] = |v_next|^2 ; sc[SC_H3] holds proj
    T H1 = sc[SC_H1], H2 = sc[SC_H2], H3 = sc[SC_H3];
    const T H4 = sqrt(out[0]);
    const int it = isc[ISC_IT] + 1;            // 1-based index of the iteration being completed
    const T c_prev = sc[SC_C_PREV], s_prev = sc[SC_S_PREV], c_curr = sc[SC_C_CURR], s_curr = sc[SC_S_CURR];
    if (it > 2) { H1 = s_prev * H2; H2 = c_prev * H2; }
    if (it > 1) {
      const T tmp = -s_curr * H2 + c_curr * H3;
      H2 = c_curr * H2 + s_curr * H3;
      H3 = tmp;
    }
    T c, s, r;
    givens_rot(H3, H4, c, s, r);
    H3 = r;
    const T rhs2 = -s * sc[SC_RHS_1];
    const T rhs1 = c * sc[SC_RHS_1];
    // coefficients for the vector update of this iteration
    sc[SC_K3_INV_H4] = T(1) / H4;
    sc[SC_K3_H2] = H2;
    sc[SC_K3_H1] = (it > 2) ? H1 : T(0);
    sc[SC_K3_INV_H3] = T(1) / H3;
    sc[SC_K3_RHS1] = rhs1;
    // move on
    sc[SC_C_PREV] = c_curr; sc[SC_S_PREV] = s_curr; sc[SC_C_CURR] = c; sc[SC_S_CURR] = s;
    sc[SC_RHS_1] = rhs2; sc[SC_RHS_2] = rhs2;
    sc[SC_H1] = H1; sc[SC_H2] = H4; sc[SC_H3] = H3; sc[SC_H4] = H4;
    const T resnorm = tabs(rhs2);
    sc[SC_RES] = resnorm;
    isc[ISC_IT] = it;
    isc[ISC_DONE] = (resnorm <= sc[SC_TOL] || it >= isc[ISC_MAXIT]) ? 1 : 0;
  }
};

// v_next -= proj v_curr ; |v_next|^2 ; scalar recurrences in the epilogue
template <typename T>
__global__ void __launch_bounds__(kBlock) minres_lanczos2_kernel(int L, const T* __restrict__ v_curr, T* __restrict__ v_next,
                                                                 const T* __restrict__ sc, const int* __restrict__ isc,
                                                                 RedBuf<T> rb, MinresStepFin<T> fin) {
  if (isc[ISC_DONE]) return;
  const T proj = sc[SC_H3];
  T accS[1] = {0};
  T accM[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    const T v = v_next[i] - proj * v_curr[i];
    v_next[i] = v;
    accS[0] += v * v;
  }
  reduce_and_finalize<T, 1, 0>(accS, accM, rb, fin);
}

// v_next /= H[4] ; w_next = (v_curr - H[2] w_curr - H[1] w_prev) / H[3] ; x += rhs[1] w_next
// Runs iff iteration `it_host` was completed on the device (also for the iteration that set done).
template <typename T>
__global__ void __launch_bounds__(kBlock) minres_update_kernel(int L, int it_host, const T* __restrict__ v_curr,
                                                               T* __restrict__ v_next, const T* __restrict__ w_prev,
                                                               const T* __restrict__ w_curr, T* __restrict__ w_next,
                                                               T* __restrict__ x, const T* __restrict__ sc,
                                                               const int* __restrict__ isc) {
  if (isc[ISC_IT] < it_host) return;
  const T inv_h4 = sc[SC_K3_INV_H4], h2 = sc[SC_K3_H2], h1 = sc[SC_K3_H1], inv_h3 = sc[SC_K3_INV_H3], rhs1 = sc[SC_K3_RHS1];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    v_next[i] *= inv_h4;
    const T w = (v_curr[i] - h2 * w_curr[i] - h1 * w_prev[i]) * inv_h3;
    w_next[i] = w;
    x[i] += rhs1 * w;
  }
}

// elementwise ADMM tail for solvers that return nu directly (full-KKT MINRES):
//   s_tl = 2 s - w_s - nu ./ rho ; w_s += alpha (s_tl - s)         (solver.jl:55,64)
template <typename T>
__global__ void __launch_bounds__(kBlock) admm_tail_kernel(int m, const T* __restrict__ nu, const T* __restrict__ rho,
                                                           const T* __restrict__ s, const T* ws_in,
                                                           T* ws_out, T alpha) {   // ws_in may alias ws_out (after a rho adaptation)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const T sr = s[i], w = ws_in[i];
    const T s_tl = T(2) * sr - w - nu[i] / rho[i];
    ws_out[i] = w + alpha * (s_tl - sr);
  }
}

// update!(q=, b=) from the model's own fp64 values, as the host scales them: q_out = T((D q') c) with q' = [q; 0] (q has
// n_src <= n entries) and, unless b is null, b_out = T(E b); D, E null: identity.  One rounding to T per entry.
template <typename T>
__global__ void __launch_bounds__(kBlock) scale_original_qb_kernel(long long n, long long n_src, const double* __restrict__ q,
                                                                   const T* __restrict__ D, double c, T* __restrict__ q_out,
                                                                   long long m, const double* __restrict__ b,
                                                                   const T* __restrict__ E, T* __restrict__ b_out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n + m; i += (long long)gridDim.x * blockDim.x) {
    if (i < n) {
      const double v = i < n_src ? q[i] : 0.0;
      q_out[i] = T(((D ? (double)D[i] : 1.0) * v) * c);
    } else {
      const long long r = i - n;
      b_out[r] = T((E ? (double)E[r] : 1.0) * b[r]);
    }
  }
}

// reverse_scaling! then scale_variables! of the resident iterates, in fp64 (scaling.jl:118-123,170-179):
// x = (D x) / D, s = E (s / E), mu = (((E mu) / c) / E) c; D, E null: identity
template <typename T>
__global__ void __launch_bounds__(kBlock) rescale_iterates_kernel(long long n, long long m, const T* __restrict__ D,
                                                                  const T* __restrict__ E, double c, T* __restrict__ x,
                                                                  T* __restrict__ s, T* __restrict__ mu) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n + m; i += (long long)gridDim.x * blockDim.x) {
    if (i < n) {
      const double d = D ? (double)D[i] : 1.0;
      x[i] = T((d * (double)x[i]) / d);
    } else {
      const long long r = i - n;
      const double e = E ? (double)E[r] : 1.0;
      s[r] = T(e * ((double)s[r] / e));
      mu[r] = T((((e * (double)mu[r]) / c) / e) * c);
    }
  }
}

}  // namespace cosmo
