// psd_tc.cuh -- projection of a large symmetric matrix onto the PSD cone on the tensor cores.
//
// Replaces dsyevr + clamp + syrk of the reference (convexset.jl:163-189, 219-263) for cones with N > kPsdSmallMax:
//
//     Pi_+(X) = (X + sign(X) X) / 2,      sign(X) by the scaled Newton-Schulz iteration
//     S <- gamma S;  S <- S (3 I - S^2) / 2,    gamma = alpha / u,
//         u     = min(1, |S^2|_F^(1/2)) >= rho(S)        (rigorous, a by-product of the product S^2)
//         alpha = min(alpha_max, (3 / (1 + l + l^2))^(1/2))   (minimax cubic for a spectrum in [l, 1]; l <- g(alpha l))
//     alpha_max = 1.5: the uncapped minimax scaling (alpha -> sqrt 3) folds the top of the spectrum down onto the
//     bottom, which brings eigenvalues of opposite sign and large weight close together and amplifies the rounding
//     errors of the products by 1 / l; with the cap the top never drops below g(1.5) = 0.56 while small eigenvalues
//     still grow by 2.25 per step (plain Newton-Schulz: 1.5) -- measured: two more steps, 10x smaller error.
//
// Every step is two products of commuting symmetric matrices, evaluated by tc::OzakiGemm (int8 slices on wgmma,
// exact int32 accumulation in registers, fp64 Horner epilogue): Y = S S with fused |Y|_F^2 and |I - Y|_F^2, then
// S' = c1 S + c0 (S Y).  The iteration keeps the sign of every eigenvalue because gamma rho(S) <= alpha < sqrt 3.
// Eigenvalues that are numerically zero never reach +-1 and do not have to (they enter the projection with weight
// |lambda|): once the unweighted measure delta = rms(1 - s_i^2) stalls, the weighted residual
// |S (S X) - X|_F / |X|_F -- twice an upper bound of the projection error -- decides.
// A NaN, no convergence within the cap or a workspace that does not fit in memory returns false and the caller falls
// back to the block-Jacobi eigensolver; CUDA failures throw.
#pragma once
#include "tc_gemm.cuh"

namespace cosmo {

// state[0..2] = coefficients of the update product, state[3] = l, state[4] = delta, state[5] = |Y|_F^2, state[6] = gamma,
// state[7] = alpha_max
template <int DUMMY = 0>
__global__ void ns_coef_kernel(const double* __restrict__ partial, int ntiles, int N, double* __restrict__ state) {
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  // one warp folds the per-tile partials in a fixed order (lane-strided sums, then a shuffle tree): deterministic
  double f = 0.0, d = 0.0;
  for (int i = threadIdx.x; i < ntiles; i += 32) { f += partial[2 * i]; d += partial[2 * i + 1]; }
  for (int o = 16; o > 0; o >>= 1) {
    f += __shfl_xor_sync(0xffffffffu, f, o);
    d += __shfl_xor_sync(0xffffffffu, d, o);
  }
  if (threadIdx.x != 0) return;
  double l = state[3];
  double gamma = 1.0;
  if (!(f > 0.0)) {            // zero matrix (f == 0) or NaN: hand it to the host through delta
    state[4] = (f == 0.0) ? 0.0 : f;
  } else {
    const double beta = sqrt(sqrt(f));                     // rho(S)^2 = rho(Y) <= |Y|_F
    const double u = beta < 1.0 ? beta : 1.0;
    double alpha = sqrt(3.0 / (1.0 + l + l * l));          // minimax cubic for a spectrum in [l, 1] ...
    if (alpha > state[7]) alpha = state[7];                // ... capped: see the header
    gamma = alpha / u;
    const double y = alpha * l, ya = alpha;
    const double gl = 0.5 * y * (3.0 - y * y), gu = 0.5 * ya * (3.0 - ya * ya);
    l = gl < gu ? gl : gu;
    if (l > 1.0) l = 1.0;
    state[4] = (beta < 1.0) ? 2.0 : sqrt(d / (double)N);   // the measure is void while the bound still tightens
  }
  state[0] = -0.5 * gamma * gamma * gamma;
  state[1] = 1.5 * gamma;
  state[2] = 0.0;
  state[3] = l;
  state[5] = f;
  state[6] = gamma;
}

// state[4] = |X - S W|_F / |X|_F
template <int DUMMY = 0>
__global__ void ns_residual_kernel(const double* __restrict__ partial, int ntiles, const double* __restrict__ x2, double* __restrict__ state) {
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  double r = 0.0;
  for (int i = threadIdx.x; i < ntiles; i += 32) r += partial[2 * i + 1];
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  if (threadIdx.x != 0) return;
  state[4] = (*x2 > 0.0) ? sqrt(r / *x2) : 0.0;
}

// x2[0] = |X|_F^2: one block folds the load kernel's partial sums in a fixed order
template <typename T>
__global__ void __launch_bounds__(kBlock) ns_norm_kernel(const T* __restrict__ fro_partials, int nparts, double* __restrict__ x2) {
  __shared__ double red[kWarpsPerBlock];
  double f = 0.0;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) f += (double)fro_partials[i];
  for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(0xffffffffu, f, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = f;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kWarpsPerBlock; ++w) t += red[w];
    *x2 = t;
  }
}

// S = X / |X|_F (fp64, whatever the model type); Xd: fp64 copy of X when the model type is not fp64
template <typename T>
__global__ void __launch_bounds__(kBlock) ns_scale_kernel(int N, const T* __restrict__ X, double* __restrict__ S, double* __restrict__ Xd,
                                                          const double* __restrict__ x2) {
  const double f = *x2;
  const double sc = (f > 0.0) ? 1.0 / sqrt(f) : 0.0;
  const long long total = (long long)N * N;
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
    const double x = (double)X[k];
    S[k] = x * sc;
    if (Xd) Xd[k] = x;
  }
}

// s[cone] = svec / square layout of the symmetric matrix P (already (X + sign(X) X) / 2)
template <typename T>
__global__ void __launch_bounds__(kBlock) ns_store_kernel(PsdConeDesc d, const double* __restrict__ P, T* __restrict__ s) {
  const int N = d.N;
  const double sqrt2 = 1.41421356237309504880;
  const long long total = (long long)N * N;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % N), j = (int)(e / N);
    if (i > j) continue;
    const double v = P[e];
    if (d.triangle) {
      s[d.off + svec_pos(i, j)] = (T)((i == j) ? v : sqrt2 * v);
    } else {
      s[d.off + (long long)j * N + i] = (T)v;
      s[d.off + (long long)i * N + j] = (T)v;   // mirror, convexset.jl:316-318
    }
  }
}

// W = 2 P - X  (the candidate S X recovered from P = (X + S X) / 2)
template <int DUMMY = 0>
__global__ void __launch_bounds__(kBlock) ns_w_from_p_kernel(long long total, const double* __restrict__ P, const double* __restrict__ X,
                                                             double* __restrict__ W) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x)
    W[k] = 2.0 * P[k] - X[k];
}

template <typename T>
struct PsdTc {
  tc::OzakiGemm<double> gemm;     // the iteration runs in fp64 for every model type (fp32 iterates would cost accuracy, not time)
  tc::Sliced slS, slY, slX;
  DevBuf<double> S0_d, S1_d, U_d, Xd_d, state_d, partial_d, const_d, x2_d;
  PinnedBuf<double> state_h;
  int capN = 0, shapeN = 0;
  int last_steps = 0, last_checks = 0, last_phases = 0;
  double last_delta = 0, last_resid = -1;
  // Lower end of the spectrum the scaling schedule is laid out for, adapted from call to call (ADMM iterates move
  // slowly).  A schedule for l0 takes sched_len(l0) steps; eigenvalues below l0 lag behind at the plain Newton-Schulz
  // rate, so a projection that needed more than sched_len + 6 steps was laid out too optimistically (l0 /= 10 and that
  // value is not tried again for 25 projections), one that finished on schedule lets every 2nd call probe l0 * 10.
  // Measured on config C4 (N = 2000): 24 / 21 / 19 / 22 / 25 steps for l0 = 1e-7 / 1e-6 / 1e-5 / 1e-4 / 1e-3.
  double l0_cur = 1e-7, l0_cap = 1e-2;
  int cap_hold = 0, good_streak = 0;
  static int sched_len(double l, double alpha_max) {
    int k = 0;
    while (l <= 0.999 && k < 200) {
      double a = std::sqrt(3.0 / (1.0 + l + l * l));
      if (a > alpha_max) a = alpha_max;
      const double y = a * l, gl = 0.5 * y * (3.0 - y * y), gu = 0.5 * a * (3.0 - a * a);
      l = gl < gu ? gl : gu;
      ++k;
    }
    return k;
  }
  bool configured = false;

  static int env_int(const char* name, int def) {
    const char* e = getenv(name);
    return (e && *e) ? atoi(e) : def;
  }
  // COSMO_B200_PSD_TC=0 switches the tensor-core path off (block Jacobi for every large cone)
  static bool enabled() {
    const char* e = getenv("COSMO_B200_PSD_TC");
    return !(e && e[0] == '0');
  }
  // the projection is left to block Jacobi
  static bool fall_back(const char* why) {
    if (getenv("COSMO_B200_PSD_DEBUG")) fprintf(stderr, "[psd-tc] fallback to block Jacobi: %s\n", why);
    return false;
  }

  void ensure(int N, cudaStream_t st) {
    if (!configured) {
      // fp64 model: 8 slices, 10 groups (products exact to ~2^-56 of the row maxima); fp32 model: 6 slices, 8 groups (2^-42)
      gemm.configure(sizeof(T) == 8 ? 8 : 6, sizeof(T) == 8 ? 10 : 8);
      state_d.alloc(8, false); const_d.alloc(8, false); x2_d.alloc(1, false);
      state_h.alloc(8);
      const double c[8] = {1.0, 0.0, 0.0, 0.5, 0.5, 0.0, 0.0, 0.0};   // [0..2]: plain product, [3..5]: (X + S X) / 2
      const_d.upload(c, 8, st);
      CUDA_TRY(cudaStreamSynchronize(st));
      configured = true;
    }
    if (N > capN) {
      capN = 0;
      const size_t nn = (size_t)N * N;
      const int nt = (N + tc::kTile - 1) / tc::kTile;
      S0_d.alloc(nn, false); S1_d.alloc(nn, false); U_d.alloc(nn, false);
      partial_d.alloc((size_t)nt * (nt + 1), false);
      if (sizeof(T) != 8) Xd_d.alloc(nn, false);
      const int Np = nt * tc::kTile;
      slS.ensure(Np); slY.ensure(Np); slX.ensure(Np);
      capN = N;
      shapeN = 0;
    }
    if (shapeN != N) {
      gemm.set_shape(N, st);
      const int Np = gemm.Np;
      // the padding rows / columns of the slices must be zero; the shape of the cone changed, so clear everything
      slS.clear(Np, st); slY.clear(Np, st); slX.clear(Np, st);
      shapeN = N;
    }
  }

  // X_in: N x N symmetric (ld = N) of the model type, fro_partials: partial sums of |X|_F^2.  Writes the projection in
  // the layout of the cone into s_out.  false: NaN, no convergence within the step cap, or no memory for the workspace
  // (block Jacobi needs less); every other failure throws.
  bool project(const PsdConeDesc& d, const T* X_in, const T* fro_partials, int nfro, T* /*scratch*/, T* s_out, cudaStream_t st,
               long long& launches) {
    const int N = d.N;
    try {
      ensure(N, st);
    } catch (const EngineError& e) {
      if (e.code != COSMO_B200_ERR_ALLOC) throw;
      return fall_back(e.msg.c_str());
    }
    const int g = (int)std::min<long long>(((long long)N * N + kBlock - 1) / kBlock, kMaxGrid);
    const int ntiles = gemm.ntiles;
    const double l0 = l0_cur;
    const double l_rearm = 1e-3;                         // a failed check re-arms the schedule for three more decades
    const double alpha_max = 1.5;                        // see the header
    const double tol = 1e-7;                              // quadratic convergence: the step after delta < tol reaches ~delta^2
    const double rtol = sizeof(T) == 8 ? 5e-13 : 1e-7;    // accepted weighted residual
    const int cap = env_int("COSMO_B200_TC_MAX_STEPS", 80);
    const double* X_d;
    if (sizeof(T) == 8) {
      X_d = reinterpret_cast<const double*>(X_in);
      ns_norm_kernel<T><<<1, kBlock, 0, st>>>(fro_partials, nfro, x2_d.p);
      ns_scale_kernel<T><<<g, kBlock, 0, st>>>(N, X_in, S0_d.p, (double*)nullptr, x2_d.p);
    } else {
      X_d = Xd_d.p;
      ns_norm_kernel<T><<<1, kBlock, 0, st>>>(fro_partials, nfro, x2_d.p);
      ns_scale_kernel<T><<<g, kBlock, 0, st>>>(N, X_in, S0_d.p, Xd_d.p, x2_d.p);
    }
    {
      double init[8] = {0, 0, 0, l0, 2.0, 0, 1.0, alpha_max};
      memcpy(state_h.p, init, sizeof(init));
      CUDA_TRY(cudaMemcpyAsync(state_d.p, state_h.p, 8 * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    gemm.slice(X_d, slX, st);
    launches += 2;
    double* S = S0_d.p;
    double* Sn = S1_d.p;
    double prev = 1e300, resid = -1.0, prev_resid = 1e300, delta = 2.0;
    // the host has nothing to decide while the schedule is still far from its taper: those steps are enqueued without
    // reading the state back (coefficients and scalings live on the device)
    const int nosync_until = std::max(0, sched_len(l0, alpha_max) - 3);
    int it = 0, next_check = -1, checks = 0, phases = 1;
    bool have_P = false;
    for (;;) {
      gemm.slice(S, slS, st);
      gemm.gemm(slS, slS, U_d.p, nullptr, nullptr, 1, const_d.p, partial_d.p, st);        // Y = S S
      ns_coef_kernel<0><<<1, 32, 0, st>>>(partial_d.p, ntiles, N, state_d.p);
      gemm.slice(U_d.p, slY, st);
      gemm.gemm(slS, slY, Sn, S, nullptr, 0, state_d.p, nullptr, st);                    // S' = c1 S + c0 S Y
      launches += 5;
      if (phases == 1 && it + 1 < nosync_until) { std::swap(S, Sn); ++it; continue; }
      CUDA_TRY(cudaMemcpyAsync(state_h.p, state_d.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      std::swap(S, Sn);
      ++it;
      delta = state_h[4];
      if (!(delta == delta)) return fall_back("NaN");
      if (delta < tol) break;
      // the scaling schedule has run out (l ~ 1) and delta stalls: a cluster of (numerically) zero eigenvalues
      const bool schedule_done = state_h[3] > 0.999;
      if (next_check < 0 && schedule_done) next_check = it + 1;
      if ((next_check >= 0 && it >= next_check && delta > 0.9 * prev) || it >= cap) {
        gemm.slice(S, slS, st);
        gemm.gemm(slS, slX, U_d.p, X_d, nullptr, 0, const_d.p + 3, nullptr, st);           // P = (X + S X) / 2
        residual_of_candidate(X_d, Sn, st, launches);
        launches += 2;
        CUDA_TRY(cudaMemcpyAsync(state_h.p, state_d.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        resid = state_h[4];
        ++checks;
        if (!(resid == resid)) return fall_back("NaN");
        // accept: below the tolerance, or within 100x of it and no longer improving (the floor of the arithmetic)
        if (resid < rtol || (resid < 1e2 * rtol && resid > 0.5 * prev_resid)) { have_P = true; break; }
        if (it >= cap) return fall_back("no convergence");
        prev_resid = resid;
        // eigenvalues below the schedule's range are still on their way: run the aggressive schedule again from l_rearm
        // (the converged part of the spectrum bounces inside [0.56, 1] meanwhile and settles in the taper)
        state_h[3] = l_rearm;
        CUDA_TRY(cudaMemcpyAsync(state_d.p + 3, state_h.p + 3, sizeof(double), cudaMemcpyHostToDevice, st));
        ++phases;
        next_check = -1;
      }
      prev = delta;
    }
    last_steps = it; last_checks = checks; last_delta = delta; last_resid = resid; last_phases = phases;
    const bool on_schedule = (phases == 1) && it <= sched_len(l0, alpha_max) + 6;
    if (on_schedule) {
      if (cap_hold > 0 && --cap_hold == 0) l0_cap = 1e-2;
      if (++good_streak >= 2) { good_streak = 0; l0_cur = std::min(l0 * 10.0, l0_cap); }
    } else {
      good_streak = 0;
      l0_cap = std::max(l0 * 0.1, 1e-12);                // this optimism failed: stay below it for the next 25 projections
      cap_hold = 25;
      l0_cur = std::max(l0 * (phases > 1 ? 1e-2 : 0.1), 1e-12);
    }
    if (!have_P) {
      gemm.slice(S, slS, st);
      gemm.gemm(slS, slX, U_d.p, X_d, nullptr, 0, const_d.p + 3, nullptr, st);
      launches += 2;
    }
    if (d.triangle == 2) psd_embedding_store_kernel<T, double><<<g, kBlock, 0, st>>>(d, U_d.p, s_out);
    else ns_store_kernel<T><<<g, kBlock, 0, st>>>(d, U_d.p, s_out);
    ++launches;
    if (getenv("COSMO_B200_PSD_DEBUG"))
      fprintf(stderr, "[psd-tc] N=%d steps=%d checks=%d phases=%d delta=%g resid=%g l0=%g next l0=%g\n", N, it, checks, phases, delta,
              resid, l0, l0_cur);
    CUDA_TRY(cudaGetLastError());
    return true;
  }

  // state[4] <- |S W - X|_F / |X|_F with W = 2 P - X, P in U_d, S sliced in slS.  Wbuf: scratch N x N.
  void residual_of_candidate(const double* X_d, double* Wbuf, cudaStream_t st, long long& launches) {
    const int N = gemm.N;
    const int g = (int)std::min<long long>(((long long)N * N + kBlock - 1) / kBlock, kMaxGrid);
    ns_w_from_p_kernel<0><<<g, kBlock, 0, st>>>((long long)N * N, U_d.p, X_d, Wbuf);
    gemm.slice(Wbuf, slY, st);
    gemm.gemm(slS, slY, nullptr, nullptr, X_d, 0, const_d.p, partial_d.p, st);
    ns_residual_kernel<0><<<1, 32, 0, st>>>(partial_d.p, gemm.ntiles, x2_d.p, state_d.p);
    launches += 4;
  }
};

}  // namespace cosmo
