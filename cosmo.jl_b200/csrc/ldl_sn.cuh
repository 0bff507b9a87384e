// ldl_sn.cuh -- supernodal LDL' of the quasi-definite KKT matrix K = [P + sigma I, A'; A, -diag(1/rho)] on the device,
// the counterpart of the reference's Pardiso plugins (kktsolver_pardiso.jl).  The host analysis (ldl_sn_symbolic.h)
// groups columns into supernodes, each a dense column-major panel; these kernels do everything numeric:
//
//   sn_assemble_kernel     K's values from the resident P_, At_, rho_vec_ and sigma straight into the (zeroed) panels
//   sn_small_kernel        one CTA per supernode, panel in shared memory: the descendant updates in ascending order,
//                          then the dense LDL' of the panel (diagonal block and L21 = A21 L11^-T D^-1)
//   sn_tile_update_kernel  a supernode too large for one CTA: one CTA per (output tile, group of descendants) sums its
//   sn_tile_reduce_kernel  group's updates; the groups are then subtracted in group order
//   sn_diag_kernel         blocked over launches of kTile columns: one CTA factors the kTile-wide diagonal block,
//   sn_panel_kernel        then (next launch) each CTA solves its rows of the panel below it, and
//   sn_trail_kernel        the trailing panel update runs one CTA per tile
//   sn_gather_kernel       forward solve, one warp per row of a level: the rows' gather from the solved columns
//   sn_fdiag_kernel        forward solve, one CTA per supernode: the unit-lower solve of the diagonal block
//   sn_backward_kernel     backward solve, one CTA per supernode of a depth: panel dot products, the upper solve of
//                          the diagonal block and the scatter into (y1, y2)
//
// Every sum runs in a fixed order and nothing uses floating-point atomics, so a factorisation and a solve are bitwise
// reproducible.  Products run on FMAs: fp32 stays off TF32 for accuracy, and fp64 has not been moved to DMMA (DESIGN).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "ldl.cuh"
#include "ldl_sn_symbolic.h"

namespace cosmo {
namespace sn {

constexpr int kTile = 32;                  // tiled path: output tile edge and block-column width
constexpr int kPanelThreads = 128;         // threads (= panel rows) per CTA of sn_panel_kernel
constexpr int kSmallBytes = 64 * 1024;     // panels whose shared-memory image fits take the small path

template <typename T>
struct Args {
  const int* sptr; const int64_t* rptr; const int* rows; const int64_t* off;
  const int64_t* uptr; const int* ud; const int* up0; const int* up1;
  T* Lx; T* D; T* Dinv;
  int* flags;   // [0] positive pivots, [1] zero or non-finite pivots
};

// first position in r[0, n) holding a value >= v
__device__ __forceinline__ int lower_bound(const int* r, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (r[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

template <typename T>
__device__ __forceinline__ void record_pivot(const Args<T>& a, int col, T dj) {
  a.D[col] = dj;
  a.Dinv[col] = T(1) / dj;
  if (dj > T(0)) atomicAdd(a.flags, 1);
  if (!(dj != T(0)) || !isfinite(dj)) atomicAdd(a.flags + 1, 1);
}

template <typename T>
__global__ void sn_assemble_kernel(int64_t nnz, const int64_t* __restrict__ Ksp, const int64_t* __restrict__ Ksrc,
                                   const int64_t* __restrict__ Kpos, const T* __restrict__ Pval, const T* __restrict__ Atval,
                                   const T* __restrict__ rho, T sigma, T* __restrict__ Lx) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
    Lx[Kpos[e]] = ldl_entry_value(e, Ksp, Ksrc, Pval, Atval, rho, sigma);
}

// Dense LDL' without pivoting of the h x w column-major panel F (leading dimension h) in shared memory: column j's D,
// L(j+1:h, j) = F(j+1:h, j) / d_j, then the rank-1 update of the columns right of j.  Pivots go to columns c0 + j.
template <typename T>
__device__ void panel_ldl(const Args<T>& a, T* F, int h, int w, int c0) {
  const int tid = threadIdx.x;
  for (int j = 0; j < w; ++j) {
    const T dj = F[j + h * j];
    const T inv = T(1) / dj;
    for (int i = j + 1 + tid; i < h; i += blockDim.x) F[i + h * j] *= inv;
    __syncthreads();
    const int nr = h - j - 1, nc = w - j - 1;
    for (int t = tid; t < nr * nc; t += blockDim.x) {
      const int kk = t / nr, ii = t - kk * nr;
      if (ii < kk) continue;
      const int i = j + 1 + ii, k = j + 1 + kk;
      F[i + h * k] -= F[i + h * j] * dj * F[k + h * j];
    }
    if (tid == 0) record_pivot(a, c0 + j, dj);
    __syncthreads();
  }
}

// Small path: supernodes list[0, cnt), one CTA each.  Shared memory: the h x w panel, then h ints of relative rows.
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_small_kernel(Args<T> a, const int* __restrict__ list, int cnt) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x;
  for (int c = blockIdx.x; c < cnt; c += gridDim.x) {
    const int s = list[c];
    const int c0 = a.sptr[s], w = a.sptr[s + 1] - c0;
    const int h = (int)(a.rptr[s + 1] - a.rptr[s]);
    const int* R = a.rows + a.rptr[s];
    T* F = reinterpret_cast<T*>(smem);
    int* rel = reinterpret_cast<int*>(F + (size_t)h * w);
    T* G = a.Lx + a.off[s];
    for (int t = tid; t < h * w; t += blockDim.x) F[t] = G[t];
    __syncthreads();
    for (int64_t u = a.uptr[s]; u < a.uptr[s + 1]; ++u) {
      const int d = a.ud[u], p0 = a.up0[u], p1 = a.up1[u];
      const int dc0 = a.sptr[d], wd = a.sptr[d + 1] - dc0;
      const int hd = (int)(a.rptr[d + 1] - a.rptr[d]);
      const int* Rd = a.rows + a.rptr[d];
      const T* Ld = a.Lx + a.off[d];
      const T* Dd = a.D + dc0;
      const int ni = hd - p0, nj = p1 - p0;
      for (int t = tid; t < ni; t += blockDim.x) rel[t] = lower_bound(R, h, Rd[p0 + t]);
      __syncthreads();
      for (int t = tid; t < ni * nj; t += blockDim.x) {
        const int jj = t / ni, ii = t - jj * ni;
        if (ii < jj) continue;
        T acc = T(0);
        for (int k = 0; k < wd; ++k) acc += Ld[p0 + ii + (int64_t)hd * k] * Dd[k] * Ld[p0 + jj + (int64_t)hd * k];
        F[rel[ii] + h * rel[jj]] -= acc;
      }
      __syncthreads();
    }
    panel_ldl(a, F, h, w, c0);
    for (int t = tid; t < h * w; t += blockDim.x) G[t] = F[t];
    __syncthreads();
  }
}

// (bi, bj) of lower tile t of a grid of nrt x nct tiles (bi >= bj), column-major over the lower tiles
__device__ __forceinline__ void lower_tile(int t, int nrt, int& bi, int& bj) {
  bj = 0;
  while (t >= nrt - bj) { t -= nrt - bj; ++bj; }
  bi = bj + t;
}

// Tiled path, descendant updates of one supernode (columns [c0, c0 + w), h rows R, panel F): CTA (t, g) sums the
// updates [u0 + g*chunk, u0 + (g+1)*chunk) ∩ [u0, u1) that land in lower tile t, in ascending order, into part[g].
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_tile_update_kernel(Args<T> a, int c0, int w, int h, const int* __restrict__ R,
                                                                int64_t u0, int64_t u1, int64_t chunk, T* __restrict__ part) {
  __shared__ T acc[kTile * kTile];
  __shared__ int rel[kTile];
  __shared__ int rng[4];
  const int tid = threadIdx.x;
  const int nrt = (h + kTile - 1) / kTile;
  int bi, bj;
  lower_tile(blockIdx.x, nrt, bi, bj);
  const int r0 = bi * kTile, r1 = min(h, r0 + kTile), q0 = bj * kTile, q1 = min(w, q0 + kTile);
  for (int t = tid; t < kTile * kTile; t += blockDim.x) acc[t] = T(0);
  const int64_t ub = u0 + blockIdx.y * chunk, ue = min(u1, ub + chunk);
  for (int64_t u = ub; u < ue; ++u) {
    const int d = a.ud[u], p0 = a.up0[u], p1 = a.up1[u];
    const int dc0 = a.sptr[d], wd = a.sptr[d + 1] - dc0;
    const int hd = (int)(a.rptr[d + 1] - a.rptr[d]);
    const int* Rd = a.rows + a.rptr[d];
    if (tid == 0) {   // rows of d in the tile's rows, columns of d in the tile's columns: contiguous, both ascending
      rng[0] = p0 + lower_bound(Rd + p0, hd - p0, R[r0]);
      rng[1] = p0 + lower_bound(Rd + p0, hd - p0, R[r1 - 1] + 1);
      rng[2] = p0 + lower_bound(Rd + p0, p1 - p0, c0 + q0);
      rng[3] = p0 + lower_bound(Rd + p0, p1 - p0, c0 + q1);
    }
    __syncthreads();
    const int i0 = rng[0], ni = rng[1] - rng[0], j0 = rng[2], nj = rng[3] - rng[2];
    if (ni > 0 && nj > 0) {
      for (int t = tid; t < ni; t += blockDim.x) rel[t] = lower_bound(R + r0, r1 - r0, Rd[i0 + t]);
      __syncthreads();
      const T* Ld = a.Lx + a.off[d];
      const T* Dd = a.D + dc0;
      for (int t = tid; t < ni * nj; t += blockDim.x) {
        const int jj = t / ni, ii = t - jj * ni;
        const int ti = rel[ii], tj = Rd[j0 + jj] - c0 - q0;
        if (r0 + ti < q0 + tj) continue;
        T s = T(0);
        for (int k = 0; k < wd; ++k) s += Ld[i0 + ii + (int64_t)hd * k] * Dd[k] * Ld[j0 + jj + (int64_t)hd * k];
        acc[ti + kTile * tj] += s;
      }
    }
    __syncthreads();
  }
  T* P = part + (int64_t)blockIdx.y * h * w;
  for (int t = tid; t < kTile * kTile; t += blockDim.x) {
    const int ti = t % kTile, tj = t / kTile;
    if (r0 + ti < r1 && q0 + tj < q1) P[r0 + ti + (int64_t)h * (q0 + tj)] = acc[t];
  }
}

// F -= sum over groups g = 0, 1, ... of part[g], on the lower entries of the h x w panel
template <typename T>
__global__ void sn_tile_reduce_kernel(T* __restrict__ F, const T* __restrict__ part, int groups, int h, int w) {
  const int64_t hw = (int64_t)h * w;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < hw; e += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(e % h), j = (int)(e / h);
    if (i < j) continue;
    T s = part[e];
    for (int g = 1; g < groups; ++g) s += part[g * hw + e];
    F[e] -= s;
  }
}

// Block column [b0, b0 + nb) of the panel F (h x w, columns c0 + ...), step 1: one CTA factors the nb x nb diagonal
// block in shared memory, writes D and L11 back in place and records the pivots.
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_diag_kernel(Args<T> a, T* F, int c0, int h, int b0, int nb) {
  __shared__ T Dg[kTile * kTile];
  const int tid = threadIdx.x;
  for (int t = tid; t < nb * nb; t += blockDim.x) Dg[t] = F[b0 + t % nb + (int64_t)h * (b0 + t / nb)];
  __syncthreads();
  panel_ldl(a, Dg, nb, nb, c0 + b0);
  for (int t = tid; t < nb * nb; t += blockDim.x)
    if (t % nb >= t / nb) F[b0 + t % nb + (int64_t)h * (b0 + t / nb)] = Dg[t];
}

// Step 2, in a later launch than step 1, so that every CTA reads the factored block: thread t of CTA k solves row
// b0 + nb + k * kPanelThreads + t of the panel below it, L(i, j) = (F(i, j) - sum_{k<j} L(i, k) d_k L(j, k)) / d_j.
// The CTAs write only their own rows, which no other CTA of the launch reads.
template <typename T>
__global__ void __launch_bounds__(kPanelThreads) sn_panel_kernel(T* F, int h, int b0, int nb) {
  __shared__ T Dg[kTile * kTile];
  __shared__ T row[kTile * kPanelThreads];
  const int tid = threadIdx.x;
  for (int t = tid; t < kTile * kTile; t += blockDim.x) {
    const int i = t % kTile, j = t / kTile;
    Dg[t] = (i >= j && i < nb) ? F[b0 + i + (int64_t)h * (b0 + j)] : T(0);
  }
  __syncthreads();
  const int i = b0 + nb + blockIdx.x * kPanelThreads + tid;
  if (i >= h) return;
  T* r = row + tid;
  for (int j = 0; j < nb; ++j) r[j * kPanelThreads] = F[i + (int64_t)h * (b0 + j)];
  for (int j = 0; j < nb; ++j) {
    T v = r[j * kPanelThreads];
    for (int k = 0; k < j; ++k) v -= r[k * kPanelThreads] * Dg[k + kTile * k] * Dg[j + kTile * k];
    v *= T(1) / Dg[j + kTile * j];
    r[j * kPanelThreads] = v;
    F[i + (int64_t)h * (b0 + j)] = v;
  }
}

// Trailing update after block column [b0, b1): F(i, j) -= sum_{k in [b0, b1)} L(i, k) d_k L(j, k) for j in [b1, w),
// i in [j, h); one CTA per lower tile of that region, k ascending.
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_trail_kernel(T* F, const T* __restrict__ D, int h, int w, int b0, int b1) {
  __shared__ T Li[kTile * kTile], Lj[kTile * kTile], dk[kTile];
  const int tid = threadIdx.x, nb = b1 - b0;
  const int nrt = (h - b1 + kTile - 1) / kTile;
  int bi, bj;
  lower_tile(blockIdx.x, nrt, bi, bj);
  const int r0 = b1 + bi * kTile, q0 = b1 + bj * kTile;
  for (int t = tid; t < kTile * kTile; t += blockDim.x) {
    const int x = t % kTile, k = t / kTile;
    Li[t] = (k < nb && r0 + x < h) ? F[r0 + x + (int64_t)h * (b0 + k)] : T(0);
    Lj[t] = (k < nb && q0 + x < w) ? F[q0 + x + (int64_t)h * (b0 + k)] : T(0);
  }
  if (tid < nb) dk[tid] = D[tid];
  __syncthreads();
  for (int t = tid; t < kTile * kTile; t += blockDim.x) {
    const int x = t % kTile, y = t / kTile;
    const int i = r0 + x, j = q0 + y;
    if (i >= h || j >= w || i < j) continue;
    T s = T(0);
    for (int k = 0; k < nb; ++k) s += Li[x + kTile * k] * dk[k] * Lj[y + kTile * k];
    F[i + (int64_t)h * j] -= s;
  }
}

template <typename T>
struct SolveArgs {
  const int* sptr; const int64_t* rptr; const int* rows; const int64_t* off;
  const int64_t* gptr; const int* gd; const int* gi;
  const T* Lx; const T* Dinv; const int* perm;
  const T* rhs;      // [x1; x2] in the original order
  T* y;              // permuted work vector
  T* out1; T* out2;  // y1 (n) and y2 (m) in the original order
  int n;
};

// y_r = rhs[perm[r]] - sum over the segments (d, i) of row r of L(r, d's columns) y(d's columns), for the rows
// list[0, cnt); lanes take the segments in a fixed stride, then a fixed shuffle tree
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_gather_kernel(SolveArgs<T> a, const int* __restrict__ list, int cnt) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int c = gw; c < cnt; c += nw) {
    const int r = list[c];
    T s = T(0);
    for (int64_t g = a.gptr[r] + lane; g < a.gptr[r + 1]; g += 32) {
      const int d = a.gd[g];
      const int dc0 = a.sptr[d], wd = a.sptr[d + 1] - dc0;
      const int64_t hd = a.rptr[d + 1] - a.rptr[d];
      const T* L = a.Lx + a.off[d] + a.gi[g];
      for (int k = 0; k < wd; ++k) s += L[hd * k] * a.y[dc0 + k];
    }
    s = ldl_warp_sum(s);
    if (lane == 0) a.y[r] = a.rhs[a.perm[r]] - s;
  }
}

// unit-lower solve of the diagonal block of every supernode of list[0, cnt), one CTA each, on a copy of its part of
// y in shared memory (in_smem: max width T of dynamic shared memory) or in place in y (supernodes too wide for it)
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_fdiag_kernel(SolveArgs<T> a, const int* __restrict__ list, int cnt, bool in_smem) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x;
  for (int c = blockIdx.x; c < cnt; c += gridDim.x) {
    const int s = list[c];
    const int c0 = a.sptr[s], w = a.sptr[s + 1] - c0;
    if (w == 1) continue;
    const int64_t h = a.rptr[s + 1] - a.rptr[s];
    const T* F = a.Lx + a.off[s];
    T* z = in_smem ? reinterpret_cast<T*>(smem) : a.y + c0;
    if (in_smem)
      for (int t = tid; t < w; t += blockDim.x) z[t] = a.y[c0 + t];
    __syncthreads();
    for (int j = 0; j < w - 1; ++j) {
      const T zj = z[j];
      for (int i = j + 1 + tid; i < w; i += blockDim.x) z[i] -= F[i + h * j] * zj;
      __syncthreads();
    }
    if (in_smem)
      for (int t = tid; t < w; t += blockDim.x) a.y[c0 + t] = z[t];
    __syncthreads();
  }
}

// x = D^-1 z - L' x for the supernodes list[0, cnt), one CTA each: t_j = z_j / d_j - L(R_off, j)' x(R_off) (a warp
// per column), then the upper solve of the diagonal block from the last column; x is written in place of z and
// scattered to y1 / y2.  t lives in shared memory (in_smem, as sn_fdiag_kernel) or in place in y: the dot products
// read y only at rows outside the supernode.
template <typename T>
__global__ void __launch_bounds__(kBlock) sn_backward_kernel(SolveArgs<T> a, const int* __restrict__ list, int cnt, bool in_smem) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  for (int c = blockIdx.x; c < cnt; c += gridDim.x) {
    const int s = list[c];
    const int c0 = a.sptr[s], w = a.sptr[s + 1] - c0;
    T* t = in_smem ? reinterpret_cast<T*>(smem) : a.y + c0;
    const int64_t h = a.rptr[s + 1] - a.rptr[s];
    const int* R = a.rows + a.rptr[s];
    const T* F = a.Lx + a.off[s];
    for (int j = warp; j < w; j += nwarp) {
      T acc = T(0);
      for (int64_t i = w + lane; i < h; i += 32) acc += F[i + h * j] * a.y[R[i]];
      acc = ldl_warp_sum(acc);
      if (lane == 0) t[j] = a.y[c0 + j] * a.Dinv[c0 + j] - acc;
    }
    __syncthreads();
    for (int j = w - 1; j > 0; --j) {
      const T xj = t[j];
      for (int i = tid; i < j; i += blockDim.x) t[i] -= F[j + h * i] * xj;
      __syncthreads();
    }
    for (int j = tid; j < w; j += blockDim.x) {
      const T x = t[j];
      a.y[c0 + j] = x;
      const int o = a.perm[c0 + j];
      if (o < a.n) a.out1[o] = x;
      else a.out2[o - a.n] = x;
    }
    __syncthreads();
  }
}

// tiles (bi >= bj) of a rows x cols panel, kTile square
inline int lower_tile_count(int64_t rows, int64_t cols) {
  const int64_t nrt = (rows + kTile - 1) / kTile, nct = (cols + kTile - 1) / kTile;
  int64_t t = 0;
  for (int64_t bj = 0; bj < nct; ++bj) t += nrt - bj;
  return (int)t;
}

}  // namespace sn

// The supernodal plugin (DESIGN §3c′): the analysis of ldl_sn_symbolic.h, the choice of path per supernode, the factor
// by supernodal level and the solves by level and depth.
template <typename T>
class SnPlugin : public DirectPlugin<T> {
 public:
  explicit SnPlugin(const DirectWiring<T>& w) : DirectPlugin<T>(w, "supernodal LDL'", "supernodal LDL'") {}

  // cosmo_b200_ldl_sn_stats
  void sn_stats(int64_t* o) const {
    o[0] = S_.ns; o[1] = S_.max_width; o[2] = S_.zeros(); o[3] = S_.levels;
    o[4] = this->ready_ ? small_count_ : 0; o[5] = this->ready_ ? tiled_count_ : 0; o[6] = this->solve_nodes_;
    o[7] = (int64_t)S_.update_flops;
  }

 private:
  using DirectPlugin<T>::w_;
  struct Big { int s; int64_t groups, chunk; };
  struct Level { int small0 = 0, small1 = 0; size_t smem = 0; std::vector<Big> big; };

  void build(const std::vector<int>& Prow, const std::vector<int>& Pcol, const std::vector<int>& Arow,
             const std::vector<int>& Acol, double t0) override {
    ldl_sn::Symbolic& S = S_;
    ldl_sn::analyze(w_.n, w_.m, Prow, Pcol, Arow, Acol, S);
    this->symbolic_s_ = now_s() - t0;
    cudaStream_t st = w_.stream;
    const size_t ts = sizeof(T);
    // path per supernode: the small path when the panel and its relative rows fit one CTA's shared memory; the tiled
    // path's descendant updates split into groups of about kUpdatesPerGroup, the partial sums capped at 256 MB
    constexpr int64_t kUpdatesPerGroup = 16;
    levels_.assign(S.levels, Level());
    std::vector<int> small;
    int64_t part = 0;
    small_count_ = tiled_count_ = 0;
    for (int l = 0; l < S.levels; ++l) {
      Level& L = levels_[l];
      L.small0 = (int)small.size();
      for (int k = S.lptr[l]; k < S.lptr[l + 1]; ++k) {
        const int s = S.lcols[k];
        const int64_t h = S.height(s), w = S.width(s);
        const size_t bytes = (size_t)(h * w) * ts + (size_t)h * sizeof(int);
        if (bytes <= (size_t)sn::kSmallBytes) {
          small.push_back(s);
          L.smem = std::max(L.smem, bytes);
          ++small_count_;
        } else {
          const int64_t nu = S.uptr[s + 1] - S.uptr[s];
          int64_t g = std::max<int64_t>(1, (nu + kUpdatesPerGroup - 1) / kUpdatesPerGroup);
          g = std::max<int64_t>(1, std::min<int64_t>(g, (int64_t)((256u << 20) / (h * w * ts))));
          const int64_t chunk = std::max<int64_t>(1, (nu + g - 1) / g);
          g = std::max<int64_t>(1, (nu + chunk - 1) / chunk);
          L.big.push_back(Big{s, g, chunk});
          if (nu) part = std::max(part, g * h * w);
          ++tiled_count_;
        }
      }
      L.small1 = (int)small.size();
    }
    const int64_t N = S.N, entries = S.off.empty() ? 0 : S.off.back();
    const double need = (double)entries * ts + (double)part * ts + (double)S.rows.size() * 4 + (double)S.Kpos.size() * 16 +
                        (double)S.Ksrc.size() * 8 + (double)S.ud.size() * 12 + (double)S.gd.size() * 8 + (double)N * (3 * ts + 24);
    this->fit(need, std::to_string((long long)S.stored) + " stored entries need");
    sptr_.upload(S.sptr, st); rptr_.upload(S.rptr, st); rows_.upload(S.rows, st); off_.upload(S.off, st);
    uptr_.upload(S.uptr, st); ud_.upload(S.ud, st); up0_.upload(S.up0, st); up1_.upload(S.up1, st);
    Ksp_.upload(S.Ksp, st); Ksrc_.upload(S.Ksrc, st); Kpos_.upload(S.Kpos, st);
    gptr_.upload(S.gptr, st); gd_.upload(S.gd, st); gi_.upload(S.gi, st);
    perm_.upload(S.perm, st); small_.upload(small, st);
    lrows_.upload(S.lrows, st); lcols_.upload(S.lcols, st); bcols_.upload(S.bcols, st);
    Lx_.alloc(std::max<int64_t>(entries, 1), false);
    part_.alloc(std::max<int64_t>(part, 1), false);
    D_.alloc(std::max<int64_t>(N, 1)); Dinv_.alloc(std::max<int64_t>(N, 1)); y_.alloc(std::max<int64_t>(N, 1));
    this->sync();
    CUDA_TRY(cudaFuncSetAttribute(sn::sn_small_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sn::kSmallBytes));
    CUDA_TRY(cudaFuncSetAttribute(sn::sn_fdiag_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sn::kSmallBytes));
    CUDA_TRY(cudaFuncSetAttribute(sn::sn_backward_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sn::kSmallBytes));
  }

  // memset and assembly of the panels, then level by level the small supernodes in one launch and each tiled one in
  // its own sequence of launches
  void capture_factor(T sigma) override {
    const ldl_sn::Symbolic& S = S_;
    cudaStream_t st = w_.stream;
    sn::Args<T> a;
    a.sptr = sptr_.p; a.rptr = rptr_.p; a.rows = rows_.p; a.off = off_.p;
    a.uptr = uptr_.p; a.ud = ud_.p; a.up0 = up0_.p; a.up1 = up1_.p;
    a.Lx = Lx_.p; a.D = D_.p; a.Dinv = Dinv_.p; a.flags = this->flags_.p;
    const int64_t entries = S.off.empty() ? 0 : S.off.back();
    if (entries) CUDA_TRY(cudaMemsetAsync(Lx_.p, 0, entries * sizeof(T), st));
    if (S.nnz_K)
      sn::sn_assemble_kernel<T><<<vgrid(S.nnz_K), kBlock, 0, st>>>(S.nnz_K, Ksp_.p, Ksrc_.p, Kpos_.p, w_.P.val, w_.At.val,
                                                                   w_.rho, sigma, Lx_.p);
    for (const Level& L : levels_) {
      if (L.small1 > L.small0) {
        const int cnt = L.small1 - L.small0;
        sn::sn_small_kernel<T><<<std::min(cnt, kMaxGrid), kBlock, L.smem, st>>>(a, small_.p + L.small0, cnt);
      }
      for (const Big& B : L.big) {
        const int s = B.s, c0 = S.sptr[s], w = S.width(s), h = S.height(s);
        T* F = Lx_.p + S.off[s];
        const int64_t u0 = S.uptr[s], u1 = S.uptr[s + 1];
        if (u1 > u0) {
          sn::sn_tile_update_kernel<T><<<dim3(sn::lower_tile_count(h, w), (unsigned)B.groups), kBlock, 0, st>>>(
              a, c0, w, h, rows_.p + S.rptr[s], u0, u1, B.chunk, part_.p);
          sn::sn_tile_reduce_kernel<T><<<vgrid((int64_t)h * w), kBlock, 0, st>>>(F, part_.p, (int)B.groups, h, w);
        }
        for (int b0 = 0; b0 < w; b0 += sn::kTile) {
          const int nb = std::min(sn::kTile, w - b0), b1 = b0 + nb;
          const int rows = h - b1;
          sn::sn_diag_kernel<T><<<1, kBlock, 0, st>>>(a, F, c0, h, b0, nb);
          if (rows > 0)
            sn::sn_panel_kernel<T><<<(rows + sn::kPanelThreads - 1) / sn::kPanelThreads, sn::kPanelThreads, 0, st>>>(
                F, h, b0, nb);
          if (b1 < w)
            sn::sn_trail_kernel<T><<<sn::lower_tile_count(h - b1, w - b1), kBlock, 0, st>>>(F, D_.p + c0 + b0, h, w, b0, b1);
        }
      }
    }
  }

  // the forward solve by supernodal level, the backward solve by depth
  void capture_solve() override {
    const ldl_sn::Symbolic& S = S_;
    cudaStream_t st = w_.stream;
    sn::SolveArgs<T> a;
    a.sptr = sptr_.p; a.rptr = rptr_.p; a.rows = rows_.p; a.off = off_.p;
    a.gptr = gptr_.p; a.gd = gd_.p; a.gi = gi_.p;
    a.Lx = Lx_.p; a.Dinv = Dinv_.p; a.perm = perm_.p;
    a.rhs = w_.rhs; a.y = y_.p; a.out1 = w_.y1; a.out2 = w_.y2; a.n = w_.n;
    // the diagonal solves keep their part of y in shared memory up to kSmallBytes, wider supernodes work on y in place
    auto vec_smem = [&](int wmax) { return (size_t)wmax * sizeof(T) <= (size_t)sn::kSmallBytes ? (size_t)wmax * sizeof(T) : 0; };
    for (int l = 0; l < S.levels; ++l) {
      const int r0 = S.lrptr[l], nr = S.lrptr[l + 1] - r0, k0 = S.lptr[l], ns = S.lptr[l + 1] - k0;
      sn::sn_gather_kernel<T><<<(int)std::min<int64_t>((nr + kWarpsPerBlock - 1) / kWarpsPerBlock, kMaxGrid), kBlock, 0, st>>>(
          a, lrows_.p + r0, nr);
      if (nr > ns) {   // some supernode of the level is wider than one column
        int wmax = 1;
        for (int k = k0; k < k0 + ns; ++k) wmax = std::max(wmax, S.width(S.lcols[k]));
        const size_t sm = vec_smem(wmax);
        sn::sn_fdiag_kernel<T><<<std::min(ns, kMaxGrid), kBlock, sm, st>>>(a, lcols_.p + k0, ns, sm > 0);
      }
    }
    for (size_t l = 0; l + 1 < S.bptr.size(); ++l) {
      const int k0 = S.bptr[l], ns = S.bptr[l + 1] - k0;
      int wmax = 1;
      for (int k = k0; k < k0 + ns; ++k) wmax = std::max(wmax, S.width(S.bcols[k]));
      const size_t sm = vec_smem(wmax);
      sn::sn_backward_kernel<T><<<std::min(ns, kMaxGrid), kBlock, sm, st>>>(a, bcols_.p + k0, ns, sm > 0);
    }
  }

  // stored entries (explicit zeros included), supernodal levels
  void stats_row(double* o) const override {
    o[0] = S_.N; o[1] = (double)S_.nnz_K; o[2] = (double)S_.stored; o[3] = S_.levels;
  }

  ldl_sn::Symbolic S_;   // the analysis; the graphs are built from it
  std::vector<Level> levels_;
  int small_count_ = 0, tiled_count_ = 0;
  DevBuf<int64_t> rptr_, off_, uptr_, Ksp_, Ksrc_, Kpos_, gptr_;
  DevBuf<int> sptr_, rows_, ud_, up0_, up1_, gd_, gi_, perm_, small_, lrows_, lcols_, bcols_;
  DevBuf<T> Lx_, D_, Dinv_, part_, y_;
};

}  // namespace cosmo
