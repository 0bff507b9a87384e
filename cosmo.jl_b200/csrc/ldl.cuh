// ldl.cuh -- direct LDL' solve of the quasi-definite KKT system K [y1; y2] = [x1; x2],
// K = [P + sigma I, A'; A, -diag(1/rho)], on the device: the counterpart of the reference's QdldlKKTSolver
// (kktsolver.jl:285-320).  The symbolic analysis (ordering, elimination tree, pattern of L, level schedules) runs on
// the host (ldl_symbolic.h); these kernels do everything numeric:
//
//   ldl_assemble_kernel   values of the permuted lower triangle of K from the resident P_, At_, rho_vec_ and sigma
//   ldl_factor_kernel     left-looking column LDL', one CTA per column, one launch per level (or per run of thin levels)
//   ldl_csr_gather_kernel the row-ordered copy of L the forward solve reads
//   ldl_forward_kernel    L z = P' r, one warp per row, the gather of the right-hand side fused in
//   ldl_backward_kernel   L' x = D^-1 z, one warp per column, the scatter into (y1, y2) fused in
//
// Every sum runs in a fixed order (columns k ascending in the factorisation, a fixed lane partition and shuffle tree
// in the solves) and nothing uses floating-point atomics, so a factorisation and a solve are bitwise reproducible.
// No CTA waits on another: levels are ordered by kernel boundaries, the levels of a run by __syncthreads() inside its
// single CTA.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "host.cuh"
#include "ldl_symbolic.h"

namespace cosmo {

// the sum of the sources of entry e of K, in the order the host listed them
template <typename T>
__device__ __forceinline__ T ldl_entry_value(int64_t e, const int64_t* __restrict__ Ksp, const int64_t* __restrict__ Ksrc,
                                             const T* __restrict__ Pval, const T* __restrict__ Atval,
                                             const T* __restrict__ rho, T sigma) {
  T v = T(0);
  for (int64_t s = Ksp[e]; s < Ksp[e + 1]; ++s) {
    const int64_t code = Ksrc[s];
    const int64_t idx = code >> 2;
    switch ((int)(code & 3)) {
      case ldl::SRC_P: v += Pval[idx]; break;
      case ldl::SRC_AT: v += Atval[idx]; break;
      case ldl::SRC_RHO: v += -T(1) / rho[idx]; break;
      default: v += sigma; break;
    }
  }
  return v;
}

template <typename T>
__global__ void ldl_assemble_kernel(int64_t nnz, const int64_t* __restrict__ Ksp, const int64_t* __restrict__ Ksrc,
                                    const T* __restrict__ Pval, const T* __restrict__ Atval, const T* __restrict__ rho,
                                    T sigma, T* __restrict__ Kx) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
    Kx[e] = ldl_entry_value(e, Ksp, Ksrc, Pval, Atval, rho, sigma);
}

template <typename T>
struct LdlFactorArgs {
  const int* cols;      // columns ordered by level
  const int* lptr;      // level pointers into cols
  int l0, l1;           // levels of this launch
  const int64_t* Kp; const int* Ki; const T* Kx;   // permuted lower triangle of K (diagonal first)
  const int64_t* Lp; const int* Li; T* Lx;        // L by columns
  const int64_t* Rp; const int* Rj; const int64_t* Rmap;   // L by rows, CSR -> CSC map
  T* D; T* Dinv;
  T* ws;                // gridDim.x dense workspaces of length N, zero between columns
  int64_t N;
  int* flags;           // [0] positive pivots, [1] zero or non-finite pivots
};

// Column j: w = K(j:N, j); w -= L(j:N, k) d_k L(j, k) for every k in row j of L (ascending); d_j = w_j;
// L(j+1:N, j) = w / d_j.  The entries of column k at rows >= j start at the CSC position of L(j, k) (rows ascending),
// so row j of L lists exactly where each update starts.  Only the rows of column j are touched and then cleared.
template <typename T>
__global__ void __launch_bounds__(kBlock) ldl_factor_kernel(LdlFactorArgs<T> a) {
  // (start, end, L(j,k) d_k) of up to kBlock updates, loaded in parallel: the sequential k loop then starts each update
  // from shared memory instead of a chain of dependent global loads
  __shared__ int64_t s_p[kBlock], s_end[kBlock];
  __shared__ T s_f[kBlock];
  T* w = a.ws + (int64_t)blockIdx.x * a.N;
  const int tid = threadIdx.x;
  for (int l = a.l0; l < a.l1; ++l) {
    for (int c = a.lptr[l] + blockIdx.x; c < a.lptr[l + 1]; c += gridDim.x) {
      const int j = a.cols[c];
      for (int64_t e = a.Kp[j] + tid; e < a.Kp[j + 1]; e += blockDim.x) w[a.Ki[e]] = a.Kx[e];
      const int64_t r1 = a.Rp[j + 1];
      for (int64_t r0 = a.Rp[j]; r0 < r1; r0 += kBlock) {
        if (r0 + tid < r1) {
          const int k = a.Rj[r0 + tid];
          const int64_t p = a.Rmap[r0 + tid];
          s_p[tid] = p;
          s_end[tid] = a.Lp[k + 1];
          s_f[tid] = a.Lx[p] * a.D[k];
        }
        __syncthreads();
        const int cnt = (int)min((int64_t)kBlock, r1 - r0);
        for (int t = 0; t < cnt; ++t) {
          const T f = s_f[t];
          const int64_t end = s_end[t];
          for (int64_t q = s_p[t] + tid; q < end; q += blockDim.x) w[a.Li[q]] -= a.Lx[q] * f;
          __syncthreads();
        }
      }
      __syncthreads();
      const T dj = w[j];
      const T inv = T(1) / dj;
      for (int64_t q = a.Lp[j] + tid; q < a.Lp[j + 1]; q += blockDim.x) {
        const int i = a.Li[q];
        a.Lx[q] = w[i] * inv;
        w[i] = T(0);
      }
      __syncthreads();
      if (tid == 0) {
        w[j] = T(0);
        a.D[j] = dj;
        a.Dinv[j] = inv;
        if (dj > T(0)) atomicAdd(a.flags, 1);
        if (!(dj != T(0)) || !isfinite(dj)) atomicAdd(a.flags + 1, 1);
      }
      __syncthreads();
    }
    __syncthreads();
  }
}

template <typename T>
__global__ void ldl_csr_gather_kernel(int64_t nnz, const int64_t* __restrict__ Rmap, const T* __restrict__ Lx, T* __restrict__ Rx) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nnz; r += (int64_t)gridDim.x * blockDim.x) Rx[r] = Lx[Rmap[r]];
}

__global__ void ldl_reset_flags_kernel(int* flags) {
  if (threadIdx.x < 2) flags[threadIdx.x] = 0;
}

template <typename T>
__device__ __forceinline__ T ldl_warp_sum(T s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

template <typename T>
struct LdlSolveArgs {
  const int* cols; const int* lptr; int l0, l1;
  const int64_t* ptr; const int* idx; const T* val;   // forward: L by rows; backward: L by columns
  const T* Dinv;
  const int* perm;
  const T* rhs;      // forward: [x1; x2] in the original order
  T* y;              // permuted work vector: z after the forward solve, x after the backward solve
  T* out1; T* out2;  // backward: y1 (n) and y2 (m) in the original order
  int n;
};

// z_i = rhs[perm[i]] - sum_k L(i, k) z_k
template <typename T>
__global__ void __launch_bounds__(kBlock) ldl_forward_kernel(LdlSolveArgs<T> a) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int l = a.l0; l < a.l1; ++l) {
    for (int c = a.lptr[l] + gw; c < a.lptr[l + 1]; c += nw) {
      const int i = a.cols[c];
      T s = T(0);
      for (int64_t r = a.ptr[i] + lane; r < a.ptr[i + 1]; r += 32) s += a.val[r] * a.y[a.idx[r]];
      s = ldl_warp_sum(s);
      if (lane == 0) a.y[i] = a.rhs[a.perm[i]] - s;
    }
    __syncthreads();
  }
}

// x_j = z_j / d_j - sum_{i > j} L(i, j) x_i, written in place of z_j and scattered to y1 / y2
template <typename T>
__global__ void __launch_bounds__(kBlock) ldl_backward_kernel(LdlSolveArgs<T> a) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int l = a.l0; l < a.l1; ++l) {
    for (int c = a.lptr[l] + gw; c < a.lptr[l + 1]; c += nw) {
      const int j = a.cols[c];
      T s = T(0);
      for (int64_t q = a.ptr[j] + lane; q < a.ptr[j + 1]; q += 32) s += a.val[q] * a.y[a.idx[q]];
      s = ldl_warp_sum(s);
      if (lane == 0) {
        const T x = a.y[j] * a.Dinv[j] - s;
        a.y[j] = x;
        const int o = a.perm[j];
        if (o < a.n) a.out1[o] = x;
        else a.out2[o - a.n] = x;
      }
    }
    __syncthreads();
  }
}

// ---- the direct plugin interface ----------------------------------------------------------------------------------

// What the engine hands a plugin once.  The captured graphs hold these pointers, so they stay put for its lifetime.
template <typename T>
struct DirectWiring {
  int n = 0, m = 0, device = 0, num_sms = 0;
  cudaStream_t stream = nullptr;
  CsrView<T> P, At;   // triu(P) and A' by rows: the pattern the analysis reads, the values K is assembled from
  long long nnzP = 0, nnzAt = 0;
  const T* rho = nullptr;                                  // rho_vec_
  const T* rhs = nullptr; T *y1 = nullptr, *y2 = nullptr;  // [x1; x2] in, y1 (n) and y2 (m) out
  const int* nranks = nullptr;     // the plugins are single-GPU
  long long* launches = nullptr;   // the engine's launch counter: every graph replay adds its nodes
};

// A direct LDL' plugin for K = [P + sigma I, A'; A, -diag(1/rho)] (DESIGN §3c): host analysis and uploads on first
// use, then factor(sigma) and solve() as captured graphs, refactored before the next solve after invalidate().  A
// plugin supplies its analysis and uploads, the launches of its two graphs and its row of cosmo_b200_ldl_stats.
template <typename T>
class DirectPlugin {
 public:
  // the errors read "the <name> KKT solver", "the <name> factor" and "<factorisation> factorisation of the KKT matrix"
  DirectPlugin(const DirectWiring<T>& w, const char* name, const char* factorisation)
      : w_(w), name_(name), factorisation_(factorisation) {}
  virtual ~DirectPlugin() {}
  long long factorizations() const { return factorizations_; }
  void invalidate() { dirty_ = true; }   // the rho vector or sigma changed

  // Assemble K from the resident P, A', rho vector and sigma and factor it: one captured graph, replayed on every
  // refactorisation and recaptured for another sigma (a kernel argument).  Reads back the pivot counts (the plugin's
  // only host synchronisation).
  void factor(double sigma) {
    if (!ready_) setup();
    if (!factor_graph_ || sigma != sigma_) {
      factor_nodes_ = (int)capture_graph(factor_graph_, w_.stream, [&] {
        ldl_reset_flags_kernel<<<1, 32, 0, w_.stream>>>(flags_.p);
        capture_factor((T)sigma);
      });
      sigma_ = sigma;
    }
    int flags[2] = {0, 0};
    CUDA_TRY(cudaEventRecord(ev_[0], w_.stream));
    CUDA_TRY(cudaGraphLaunch(factor_graph_, w_.stream));
    CUDA_TRY(cudaEventRecord(ev_[1], w_.stream));
    CUDA_TRY(cudaMemcpyAsync(flags, flags_.p, sizeof(flags), cudaMemcpyDeviceToHost, w_.stream));
    sync();
    *w_.launches += factor_nodes_;
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
    factor_s_ = ms * 1e-3;
    ++factorizations_;
    if (flags[1] != 0) {
      char b[160];
      snprintf(b, sizeof(b), "%s factorisation of the KKT matrix met %d zero or non-finite pivots", factorisation_, flags[1]);
      throw EngineError{COSMO_B200_ERR_NUMERICAL, b};
    }
    // positive_inertia(ldlfact) == n (kktsolver.jl:300-303)
    if (flags[0] != w_.n) throw EngineError{COSMO_B200_ERR_INVALID, "Objective function is not convex."};
    dirty_ = false;
  }

  // [y1; y2] = K \ [x1; x2], one captured graph, after a refactorisation with sigma if the factor is dirty.  kept_factor:
  // solve with the factor in memory as it is (a polish's K~); the solve reads only the factor, the right-hand side and
  // the permutation, never sigma or the rho vector.
  void solve(double sigma, bool kept_factor) {
    if (*w_.nranks > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, std::string("the ") + name_ + " KKT solver is single-GPU"};
    if (!ready_) setup();
    if (dirty_ && !kept_factor) factor(sigma);
    if (!solve_graph_) solve_nodes_ = (int)capture_graph(solve_graph_, w_.stream, [&] { capture_solve(); });
    CUDA_TRY(cudaGraphLaunch(solve_graph_, w_.stream));
    *w_.launches += solve_nodes_;
  }

  // cosmo_b200_ldl_stats: the plugin's row (N, entries of K and of L, levels), solve launches, factorisations, seconds
  // of the last factorisation and of the analysis
  void stats(double* o) const {
    stats_row(o);
    o[4] = solve_nodes_; o[5] = (double)factorizations_; o[6] = factor_s_; o[7] = symbolic_s_;
  }

 protected:
  // the host analysis of the pattern of triu(P) and A' (CSR, downloaded from t0 on), its seconds into symbolic_s_, then
  // the fit check, uploads and device buffers; returns with the stream synchronised
  virtual void build(const std::vector<int>& Prow, const std::vector<int>& Pcol, const std::vector<int>& Arow,
                     const std::vector<int>& Acol, double t0) = 0;
  // enqueue the launches of the factor after the reset of the pivot flags, and of the solve
  virtual void capture_factor(T sigma) = 0;
  virtual void capture_solve() = 0;
  virtual void stats_row(double* o) const = 0;

  void sync() const { CUDA_TRY(cudaStreamSynchronize(w_.stream)); }
  // ERR_ALLOC "the <name> factor does not fit in device memory: <what> <need> GB, <free> GB free" unless `need` bytes
  // fit in 0.9 of the free device memory
  void fit(double need, const std::string& what) const {
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    if (need > 0.9 * (double)free_b) {
      char b[96];
      snprintf(b, sizeof(b), " %.2f GB, %.2f GB free", need * 1e-9, (double)free_b * 1e-9);
      throw EngineError{COSMO_B200_ERR_ALLOC, std::string("the ") + name_ + " factor does not fit in device memory: " + what + b};
    }
  }

  const DirectWiring<T> w_;
  bool ready_ = false;
  int solve_nodes_ = 0;
  double symbolic_s_ = 0.0;
  DevBuf<int> flags_;   // [0] positive pivots, [1] zero or non-finite pivots

 private:
  // download of the pattern, host analysis, uploads
  void setup() {
    CUDA_TRY(cudaSetDevice(w_.device));
    const double t0 = now_s();
    std::vector<int> Prow(w_.n + 1), Pcol(w_.nnzP), Arow(w_.n + 1), Acol(w_.nnzAt);
    CUDA_TRY(cudaMemcpyAsync(Prow.data(), w_.P.rowptr, (w_.n + 1) * sizeof(int), cudaMemcpyDeviceToHost, w_.stream));
    CUDA_TRY(cudaMemcpyAsync(Arow.data(), w_.At.rowptr, (w_.n + 1) * sizeof(int), cudaMemcpyDeviceToHost, w_.stream));
    if (w_.nnzP) CUDA_TRY(cudaMemcpyAsync(Pcol.data(), w_.P.col, w_.nnzP * sizeof(int), cudaMemcpyDeviceToHost, w_.stream));
    if (w_.nnzAt) CUDA_TRY(cudaMemcpyAsync(Acol.data(), w_.At.col, w_.nnzAt * sizeof(int), cudaMemcpyDeviceToHost, w_.stream));
    sync();
    build(Prow, Pcol, Arow, Acol, t0);
    flags_.alloc(2);
    ev_[0].create(); ev_[1].create();
    ready_ = dirty_ = true;
  }

  const char* name_;
  const char* factorisation_;
  bool dirty_ = true;
  double sigma_ = 0.0;   // the one factor_graph_ holds
  int factor_nodes_ = 0;
  long long factorizations_ = 0;
  double factor_s_ = 0.0;
  GraphExec factor_graph_, solve_graph_;
  Event ev_[2];
};

// The simplicial plugin (DESIGN §3c): the analysis of ldl_symbolic.h, the factor and the solves of the kernels above.
template <typename T>
class LdlPlugin : public DirectPlugin<T> {
 public:
  explicit LdlPlugin(const DirectWiring<T>& w) : DirectPlugin<T>(w, "direct LDL'", "LDL'") {}

 private:
  using DirectPlugin<T>::w_;

  void build(const std::vector<int>& Prow, const std::vector<int>& Pcol, const std::vector<int>& Arow,
             const std::vector<int>& Acol, double t0) override {
    ldl::Symbolic S;
    ldl::analyze(w_.n, w_.m, Prow, Pcol, Arow, Acol, S);
    this->symbolic_s_ = now_s() - t0;
    const int N = N_ = S.N;
    nnzK_ = S.nnz_triu_K();
    nnzL_ = S.nnz_L();
    cudaStream_t st = w_.stream;
    // one dense workspace of length N per resident factor CTA: as many CTAs as the widest level, at most two per SM
    int maxw = 1;
    for (const ldl::Segment& s : S.fseg)
      if (!s.run) maxw = std::max(maxw, S.fptr[s.l1] - S.fptr[s.l0]);
    ws_ctas_ = std::max(1, std::min(maxw, 2 * w_.num_sms));
    const double ts = (double)sizeof(T);
    const double need = (double)nnzL_ * (2 * ts + 4 + 4 + 8) + (double)nnzK_ * (ts + 4 + 8) + (double)S.Ksrc.size() * 8 +
                        (double)(N + 1) * 8 * 3 + (double)N * (ts * 3 + 4 * 5) + (double)ws_ctas_ * N * ts;
    this->fit(need, "nnz(L) = " + std::to_string(nnzL_) + " needs");
    Kp_.upload(S.Kp, st); Ki_.upload(S.Ki, st); Ksp_.upload(S.Ksp, st); Ksrc_.upload(S.Ksrc, st);
    Lp_.upload(S.Lp, st); Li_.upload(S.Li, st);
    Rp_.upload(S.Rp, st); Rj_.upload(S.Rj, st); Rmap_.upload(S.Rmap, st);
    fcols_.upload(S.fcols, st); fptr_.upload(S.fptr, st);
    bcols_.upload(S.bcols, st); bptr_.upload(S.bptr, st);
    perm_.upload(S.perm, st);
    Kx_.alloc(std::max<long long>(nnzK_, 1), false);
    Lx_.alloc(std::max<long long>(nnzL_, 1), false);
    Rx_.alloc(std::max<long long>(nnzL_, 1), false);
    D_.alloc(std::max(N, 1)); Dinv_.alloc(std::max(N, 1)); y_.alloc(std::max(N, 1));
    ws_.alloc((size_t)ws_ctas_ * std::max(N, 1));   // zeroed: every column clears what it touched
    this->sync();
    fseg_ = S.fseg; bseg_ = S.bseg;
    fptr_h_ = S.fptr; bptr_h_ = S.bptr;
  }

  void capture_factor(T sigma) override {
    cudaStream_t st = w_.stream;
    ldl_assemble_kernel<T><<<vgrid(nnzK_), kBlock, 0, st>>>(nnzK_, Ksp_.p, Ksrc_.p, w_.P.val, w_.At.val, w_.rho, sigma, Kx_.p);
    LdlFactorArgs<T> a;
    a.cols = fcols_.p; a.lptr = fptr_.p;
    a.Kp = Kp_.p; a.Ki = Ki_.p; a.Kx = Kx_.p;
    a.Lp = Lp_.p; a.Li = Li_.p; a.Lx = Lx_.p;
    a.Rp = Rp_.p; a.Rj = Rj_.p; a.Rmap = Rmap_.p;
    a.D = D_.p; a.Dinv = Dinv_.p; a.ws = ws_.p; a.N = N_; a.flags = this->flags_.p;
    for (const ldl::Segment& s : fseg_) {
      a.l0 = s.l0; a.l1 = s.l1;
      const int grid = s.run ? 1 : std::min(fptr_h_[s.l1] - fptr_h_[s.l0], ws_ctas_);
      ldl_factor_kernel<T><<<grid, kBlock, 0, st>>>(a);
    }
    if (nnzL_) ldl_csr_gather_kernel<T><<<vgrid(nnzL_), kBlock, 0, st>>>(nnzL_, Rmap_.p, Lx_.p, Rx_.p);
  }

  // forward levels, then backward depths
  void capture_solve() override {
    cudaStream_t st = w_.stream;
    LdlSolveArgs<T> a;
    a.Dinv = Dinv_.p; a.perm = perm_.p; a.rhs = w_.rhs; a.y = y_.p; a.out1 = w_.y1; a.out2 = w_.y2; a.n = w_.n;
    auto grid = [&](const std::vector<int>& ptr, const ldl::Segment& s) {
      return s.run ? 1 : (int)std::min<long long>(((long long)ptr[s.l1] - ptr[s.l0] + kWarpsPerBlock - 1) / kWarpsPerBlock, kMaxGrid);
    };
    a.cols = fcols_.p; a.lptr = fptr_.p; a.ptr = Rp_.p; a.idx = Rj_.p; a.val = Rx_.p;
    for (const ldl::Segment& s : fseg_) {
      a.l0 = s.l0; a.l1 = s.l1;
      ldl_forward_kernel<T><<<grid(fptr_h_, s), kBlock, 0, st>>>(a);
    }
    a.cols = bcols_.p; a.lptr = bptr_.p; a.ptr = Lp_.p; a.idx = Li_.p; a.val = Lx_.p;
    for (const ldl::Segment& s : bseg_) {
      a.l0 = s.l0; a.l1 = s.l1;
      ldl_backward_kernel<T><<<grid(bptr_h_, s), kBlock, 0, st>>>(a);
    }
  }

  void stats_row(double* o) const override {
    o[0] = N_; o[1] = (double)nnzK_; o[2] = (double)nnzL_; o[3] = fptr_h_.empty() ? 0 : (double)fptr_h_.size() - 1;
  }

  std::vector<ldl::Segment> fseg_, bseg_;
  std::vector<int> fptr_h_, bptr_h_;
  int N_ = 0, ws_ctas_ = 1;
  long long nnzK_ = 0, nnzL_ = 0;
  DevBuf<int64_t> Kp_, Ksp_, Ksrc_, Lp_, Rp_, Rmap_;
  DevBuf<int> Ki_, Li_, Rj_, fcols_, fptr_, bcols_, bptr_, perm_;
  DevBuf<T> Kx_, Lx_, Rx_, D_, Dinv_, ws_, y_;
};

}  // namespace cosmo
