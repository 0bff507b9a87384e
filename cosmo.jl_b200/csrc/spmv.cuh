// spmv.cuh -- CSR SpMV family with fused epilogues (kernels K1-K3 of SURVEY.md 2a).
//
// Replaces the reference's single-threaded SparseArrays.mul! calls at
//   src/linear_solver/kktsolver_indirect.jl:53,59-63,81   (KKT operator)
//   src/residuals.jl:4,12,15,65,81,91,145                  (residuals / cost)
//   src/infeasibility.jl:12,44,53                          (certificates)
//
// One kernel template serves every use: a row's dot product is taken over up
// to two CSR matrices that share the row index (A' and P for the reduced KKT
// operator  c = A'(rho.*(A u)) + P u + sigma u), then a functor epilogue turns
// (row, sum) into the output and into up to 8 deterministic reductions.
//
// HBM-bound: 12 B per nonzero (8 B value + 4 B index) are streamed once with
// 128-bit __ldcs loads (values: 2 x double2, indices: int4 per lane per step),
// the gathered vector is read through L1/L2 with __ldg.  Rows are peeled to a
// 4-element boundary so that the streams stay 16/32-byte aligned.
#pragma once
#include "common.cuh"
#include "win_pack.h"

namespace cosmo {

// Gather of the dense operand: through the read-only (non-coherent) path when the vector is constant
// for the lifetime of the kernel, through L2 (ld.global.cg) when the same kernel also writes it
// (the persistent CG kernel re-reads vectors across grid barriers).
template <typename T, bool NC>
__device__ __forceinline__ T gather_ld(const T* p) {
  if (NC) return __ldg(p);
  return __ldcg(p);
}

// Partial dot product of one CSR row with a dense vector, LANES cooperating
// lanes (32 => vectorised stream path).  Returns this lane's partial sum.
template <typename T, int LANES, bool NC = true>
__device__ __forceinline__ T row_partial(const CsrView<T>& M, const T* __restrict__ x, int row, int lane) {
  const int start = __ldg(M.rowptr + row);
  const int end = __ldg(M.rowptr + row + 1);
  T s0 = 0, s1 = 0;
  if (LANES == 32) {
    int a0 = (start + 3) & ~3;
    if (a0 > end) a0 = end;
    {  // head: < 4 unaligned elements
      const int i = start + lane;
      if (i < a0) s0 += __ldcs(M.val + i) * gather_ld<T, NC>(x + __ldcs(M.col + i));
    }
    const int body_end = a0 + ((end - a0) & ~3);
#pragma unroll 2
    for (int j = a0 + lane * 4; j < body_end; j += 128) {
      const int4 c = load4_stream(M.col + j);
      T v[4];
      load4_stream(M.val + j, v);
      s0 += v[0] * gather_ld<T, NC>(x + c.x);
      s1 += v[1] * gather_ld<T, NC>(x + c.y);
      s0 += v[2] * gather_ld<T, NC>(x + c.z);
      s1 += v[3] * gather_ld<T, NC>(x + c.w);
    }
    {  // tail: < 4 elements
      const int i = body_end + lane;
      if (i < end) s1 += __ldcs(M.val + i) * gather_ld<T, NC>(x + __ldcs(M.col + i));
    }
  } else {
    for (int j = start + lane; j < end; j += LANES) s0 += __ldcs(M.val + j) * gather_ld<T, NC>(x + __ldcs(M.col + j));
  }
  return s0 + s1;
}

template <typename T, int LANES>
__device__ __forceinline__ T group_sum(T v) {
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, LANES);
  return v;
}

// Epi concept:
//   static constexpr int NS, NM;            reduction slots (sums, maxes)
//   const int* done;                        optional early-exit flag (nullptr = none)
//   __device__ void row(int r, T sum, T* accS, T* accM) const;
//   __device__ void finalize(T* out) const; scalar epilogue, one thread, after the fold
template <typename T, int LANES, typename Epi>
__global__ void __launch_bounds__(kBlock) spmv_kernel(CsrView<T> M1, const T* __restrict__ x1, CsrView<T> M2,
                                                      const T* __restrict__ x2, int nrows, Epi epi, RedBuf<T> rb) {
  pdl_launch_dependents();
  pdl_wait();
  if (epi.done != nullptr && *epi.done) return;
  constexpr int GROUPS = kBlock / LANES;
  const int lane = threadIdx.x % LANES;
  const int group = threadIdx.x / LANES;
  const int total_groups = gridDim.x * GROUPS;
  T accS[Epi::NS > 0 ? Epi::NS : 1];
  T accM[Epi::NM > 0 ? Epi::NM : 1];
#pragma unroll
  for (int k = 0; k < (Epi::NS > 0 ? Epi::NS : 1); ++k) accS[k] = 0;
#pragma unroll
  for (int k = 0; k < (Epi::NM > 0 ? Epi::NM : 1); ++k) accM[k] = 0;

  // `base` is block-uniform so every lane of a warp runs the same number of trips:
  // the full-mask shuffles below (and in the reduction) must be reached by all 32 lanes.
  for (int base = blockIdx.x * GROUPS; base < nrows; base += total_groups) {
    const int row = base + group;
    const bool valid = row < nrows;
    T s = 0;
    if (valid) {
      if (M1.rowptr != nullptr) s += row_partial<T, LANES>(M1, x1, row, lane);
      if (M2.rowptr != nullptr) s += row_partial<T, LANES>(M2, x2, row, lane);
    }
    s = group_sum<T, LANES>(s);
    if (valid && lane == 0) epi.row(row, s, accS, accM);
  }
  if constexpr (Epi::NS + Epi::NM > 0) {
    reduce_and_finalize<T, Epi::NS, Epi::NM>(accS, accM, rb, epi);
  }
}

// ---------------------------------------------------------------------------
// Column-windowed SpMV: the gathered vector is staged in shared memory.
//
// The plain kernel above is limited by the L1TEX wavefront rate (one scattered
// 8-byte gather per cycle per SM), not by HBM.  Here the matrix is stored as
// `nwin` column slabs ("windows") of width W <= 25.6k doubles; a persistent CTA
// per SM pulls the W-slice of x into its 200 KB of shared memory with one TMA
// bulk copy (cp.async.bulk + mbarrier), then streams its rows of that slab
// from HBM and gathers from shared memory.  Rows are padded to 8 entries so
// every lane issues aligned loads; values are laid out so that each warp-wide
// load instruction covers one contiguous 512-byte run.  Partial row sums are
// carried between windows in a small global vector; the epilogue runs on the
// last window.  Two slab layouts (the PACKED template argument):
//   10 B per entry: 8-byte values + 16-bit window-local column indices.
//    9 B per entry (fp64 only, win_pack.h): an 8-byte word holding sign, a 4-bit exponent code, the low 7 column bits
//                   and the mantissa, where the value sits in the 10 B layout, and one byte of high column bits, where
//                   the column sits.  The decode is exact, so both layouts compute the same sums bit for bit.
// Streamed HBM traffic is 10 or 9 B/nnz (+1.4 % padding on C2), against 12 for plain CSR.
// ---------------------------------------------------------------------------
template <typename T>
struct WcsrView {
  const int* rowptr;            // nwin * (nrows + 1), element offsets (multiples of 8)
  const unsigned short* col;    // 10 B layout: window-local column index
  const T* val;                 // 10 B layout: value
  const unsigned long long* word;   // 9 B layout: packed words (win_pack.h)
  const unsigned char* colhi;       // 9 B layout: column bits 7-14
  const double* esc;                // 9 B layout: escaped values
  unsigned kexp;                    // 9 B layout: winpack::exp_offset(ebase)
  const int* cta_row_start;     // gridDim.x + 1 contiguous row chunks, balanced by nnz
  int nwin, W, nrows, ncols;
};

constexpr int kWinThreads = 1024;
constexpr int kWinWarps = kWinThreads / 32;

// One lane's 8 entries of a slab step, as loaded: `v` from the value (or word) stream, `c` from the column stream.
// val(i) / col(i) give entry i; the packed layout decodes it here, right before its FMA.
template <typename T, bool PACKED>
struct WinStep {
  using Col = uint4;
  T v[8];
  Col c;
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = T(0);
    c = make_uint4(0, 0, 0, 0);
  }
  __device__ __forceinline__ void load(const WcsrView<T>& M, int s, int L, int lane) {
    c = __ldcs(reinterpret_cast<const uint4*>(M.col + s + lane * 8));
    load8_coalesced(M.val + s, L, lane, v);
  }
  __device__ __forceinline__ T val(const WcsrView<T>&, int i) const { return v[i]; }
  __device__ __forceinline__ unsigned col(int i) const {
    const unsigned w = i < 2 ? c.x : i < 4 ? c.y : i < 6 ? c.z : c.w;
    return (i & 1) ? w >> 16 : w & 0xffffu;
  }
};
template <>
struct WinStep<double, true> {
  double v[8];   // packed words, loaded through the double path of load8_coalesced
  uint2 c;       // 8 column-high bytes
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.0;
    c = make_uint2(0, 0);
  }
  __device__ __forceinline__ void load(const WcsrView<double>& M, int s, int L, int lane) {
    c = __ldcs(reinterpret_cast<const uint2*>(M.colhi + s + lane * 8));
    load8_coalesced(reinterpret_cast<const double*>(M.word) + s, L, lane, v);
  }
  // an escape reads its value from the table with a predicated load, not a branch
  __device__ __forceinline__ double val(const WcsrView<double>& M, int i) const {
    const unsigned hi = (unsigned)__double2hiint(v[i]), lo = (unsigned)__double2loint(v[i]);
    double d = __hiloint2double((int)winpack::decode_hi(hi, M.kexp), (int)lo);
    if (winpack::is_escape(hi)) d = __ldg(M.esc + lo);
    return d;
  }
  __device__ __forceinline__ unsigned col(int i) const {
    const unsigned hb = __byte_perm(i < 4 ? c.x : c.y, 0u, (unsigned)(i & 3) | 0x4440u);
    return winpack::decode_col((unsigned)__double2hiint(v[i]), hb);
  }
};

__device__ __forceinline__ double win_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float win_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double win_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ float win_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }

// gather-FMA of one lane's 8 entries against the staged x slice.  The roundings are spelled out, so that both layouts
// (and every build) sum in the same order: s0 = v0 x0 + v2 x2 + v4 x4 + v6 x6 with the product v2 x2 rounded and the
// others fused, s1 likewise over the odd slots.
template <typename T, bool PACKED>
__device__ __forceinline__ T win_fma8(const WinStep<T, PACKED>& e, const WcsrView<T>& M, const T* xs) {
  T s0 = win_mul(e.val(M, 2), xs[e.col(2)]);
  T s1 = win_mul(e.val(M, 3), xs[e.col(3)]);
  s0 = win_fma(e.val(M, 0), xs[e.col(0)], s0);
  s1 = win_fma(e.val(M, 1), xs[e.col(1)], s1);
  s0 = win_fma(e.val(M, 4), xs[e.col(4)], s0);
  s1 = win_fma(e.val(M, 5), xs[e.col(5)], s1);
  s0 = win_fma(e.val(M, 6), xs[e.col(6)], s0);
  s1 = win_fma(e.val(M, 7), xs[e.col(7)], s1);
  return s0 + s1;
}

// steps beyond the first 256 entries of a row segment (long rows)
template <typename T, bool PACKED>
__device__ __forceinline__ T win_row_rest(const WcsrView<T>& M, const T* xs, int start, int end, int lane) {
  T s = 0;
  for (int j0 = start + 256; j0 < end; j0 += 256) {
    const int L = min(32, (end - j0) >> 3);
    if (lane < L) {
      WinStep<T, PACKED> e;
      e.load(M, j0, L, lane);
      s += win_fma8<T, PACKED>(e, M, xs);
    }
  }
  return s;
}

// One CTA per (row chunk j, window w): b = j * nwin + w.  The CTA stages its W-slice of x once
// (a single TMA bulk copy that overlaps the first row loads), streams the rows of chunk j in
// slab w and writes per-window partial sums.  The last of the nwin CTAs of a chunk to finish
// (per-chunk ticket) folds the partials in window order -- deterministic -- and runs the epilogue
// (one thread per row); only those "finishing" CTAs take part in the scalar reduction, whose
// partials are indexed by chunk, not by CTA.
//
// PL > 0 (the reduced KKT operator): the P-row product p = M2 x2 of chunk j's rows is spread over the nwin CTAs of the
// chunk, PL lanes per row, and stored in `pbuf`, which the epilogue reads as its `add` vector.  With nwin > 1 each CTA
// sums its share after streaming its slab, and the finishing CTA reads them after the chunk ticket; with nwin == 1
// the CTA sums them before streaming, behind a CTA barrier.  Every P row is summed exactly as
// spmv_kernel<T, PL, EpiStore> sums it (row_partial + group_sum with the same PL), so the result is bitwise that of a
// separate P launch.  PL = 0: no P rows (M2, x2 and pbuf unused).
template <typename T, bool PACKED, typename Epi, int PL = 0>
__global__ void __launch_bounds__(kWinThreads, 1) spmv_win_kernel(WcsrView<T> M, const T* __restrict__ x, CsrView<T> M2,
                                                                  const T* __restrict__ x2, Epi epi, RedBuf<T> rb,
                                                                  T* __restrict__ ypart, unsigned* __restrict__ chunk_ticket,
                                                                  T* pbuf) {
  pdl_launch_dependents();
  extern __shared__ __align__(128) unsigned char win_smem[];
  T* xs = reinterpret_cast<T*>(win_smem);
  __shared__ __align__(8) uint64_t bar;
  __shared__ int fin_flag;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int w = blockIdx.x % M.nwin, chunk = blockIdx.x / M.nwin;
  const int nchunks = gridDim.x / M.nwin;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  // Up to the first pdl_wait() (in `stage_x`) only the constant slab arrays are read: the barrier setup, the row
  // pointers and (PL = 0) the first row pair's columns and values overlap the tail of the kernel before this one.  The
  // x-slice, the done flag, x2 and every output are touched after it.  stage_x() waits, then issues the bulk copy.
  auto stage_x = [&]() -> bool {
    pdl_wait();
    if (epi.done != nullptr && *epi.done) return false;
    if (threadIdx.x == 0) {
      int cnt = M.ncols - w * M.W;
      if (cnt > M.W) cnt = M.W;
      const unsigned bytes = ((unsigned)cnt * (unsigned)sizeof(T) + 15u) & ~15u;   // source buffers are padded
      mbar_expect_tx(&bar, bytes);
      bulk_load_g2s(xs, x + (size_t)w * M.W, bytes, &bar);
    }
    return true;
  };
  const int r0 = M.cta_row_start[chunk], r1 = M.cta_row_start[chunk + 1];
  T accS[Epi::NS > 0 ? Epi::NS : 1];
  T accM[Epi::NM > 0 ? Epi::NM : 1];
#pragma unroll
  for (int k = 0; k < (Epi::NS > 0 ? Epi::NS : 1); ++k) accS[k] = 0;
#pragma unroll
  for (int k = 0; k < (Epi::NM > 0 ? Epi::NM : 1); ++k) accM[k] = 0;

  const int* rp = M.rowptr + (size_t)w * (M.nrows + 1);
  const bool single = (M.nwin == 1);
  T* yw = ypart + (size_t)w * M.nrows;
  // This warp owns rows r0 + warp + k * kWinWarps, two of them in flight at a time.  Row
  // pointers of the NEXT pair are fetched (warp-uniform loads) before the current pair is
  // consumed, so they stay off the critical path.
  const int nmine = (r1 - r0 - warp + kWinWarps - 1) / kWinWarps;   // rows of this warp (<= 0: none)
  bool waited = false;
  int sa = 0, ea = 0, sb = 0, eb = 0;
  auto fetch_ptrs = [&](int k, int& s_a, int& e_a, int& s_b, int& e_b) {
    s_a = e_a = s_b = e_b = 0;
    if (k < nmine) {
      const int row = r0 + warp + k * kWinWarps;
      s_a = __ldg(rp + row);
      e_a = __ldg(rp + row + 1);
    }
    if (k + 1 < nmine) {
      const int row = r0 + warp + (k + 1) * kWinWarps;
      s_b = __ldg(rp + row);
      e_b = __ldg(rp + row + 1);
    }
  };
  // this CTA's share of the chunk's P rows (called block-uniformly, after the wait)
  auto p_rows = [&]() {
    constexpr int G = kWinThreads / (PL > 0 ? PL : 1);
    const int plane = threadIdx.x % (PL > 0 ? PL : 1), group = threadIdx.x / (PL > 0 ? PL : 1);
    // `base` is block-uniform so every lane of a warp runs the same number of trips (full-mask shuffles)
    for (int base = r0 + w * G; base < r1; base += M.nwin * G) {
      const int row = base + group;
      const bool valid = row < r1;
      T s = 0;
      if (valid) s += row_partial<T, (PL > 0 ? PL : 1)>(M2, x2, row, plane);
      s = group_sum<T, (PL > 0 ? PL : 1)>(s);
      if (valid && plane == 0) pbuf[row] = s;
    }
  };
  fetch_ptrs(0, sa, ea, sb, eb);
  bool staged = false;
  if constexpr (PL > 0) {
    if (single) {
      // the epilogue runs in the streaming loop: wait, start the x-slice copy, sum the P rows under it, and make them
      // visible to the whole CTA before streaming
      if (!stage_x()) return;
      staged = true;
      p_rows();
      __syncthreads();
    }
  }
  for (int k = 0; k < nmine; k += 2) {
    const bool has_b = (k + 1 < nmine);
    const int ja = sa + lane * 8, jb = sb + lane * 8;
    const bool la = ja < ea, lb = jb < eb;
    WinStep<T, PACKED> stepa, stepb;
    stepa.clear();
    stepb.clear();
    if (la) stepa.load(M, sa, min(32, (ea - sa) >> 3), lane);
    if (lb) stepb.load(M, sb, min(32, (eb - sb) >> 3), lane);
    // long segments (> one 256-entry step) re-read their row pointers after the first step instead of holding them
    const bool longa = ea - sa > 256, longb = eb - sb > 256;
    fetch_ptrs(k + 2, sa, ea, sb, eb);          // next pair
    if (!waited) {
      if (!staged && !stage_x()) return;
      mbar_wait(&bar, 0);
      waited = true;
    }
    T pa = la ? win_fma8<T, PACKED>(stepa, M, xs) : T(0);
    T pb = lb ? win_fma8<T, PACKED>(stepb, M, xs) : T(0);
    const int rowa = r0 + warp + k * kWinWarps;
    const int rowb = rowa + kWinWarps;
    if (longa) pa += win_row_rest<T, PACKED>(M, xs, __ldg(rp + rowa), __ldg(rp + rowa + 1), lane);
    if (longb) pb += win_row_rest<T, PACKED>(M, xs, __ldg(rp + rowb), __ldg(rp + rowb + 1), lane);
    // paired reduction: lanes 0-15 fold row a, lanes 16-31 fold row b (5 shuffles for 2 rows)
    const bool hi = (lane & 16) != 0;
    T keep = hi ? pb : pa;
    const T send = hi ? pa : pb;
    keep += __shfl_xor_sync(0xffffffffu, send, 16);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) keep += __shfl_xor_sync(0xffffffffu, keep, o);
    if (lane == 0 || (lane == 16 && has_b)) {
      const int row = hi ? rowb : rowa;
      if (single) epi.row(row, keep, accS, accM);
      else yw[row] = keep;
    }
  }
  if (!waited) {   // warps without rows: the x-slice is still staged by thread 0, never left in flight
    if (!staged && !stage_x()) return;
    mbar_wait(&bar, 0);
  }
  // nwin > 1: the P rows fill the time between this CTA's last row and the chunk ticket; the finishing CTA reads them
  // after the ticket's fences
  if constexpr (PL > 0) {
    if (!single) p_rows();
  }

  if (!single) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned t = atomicAdd(chunk_ticket + chunk, 1u);
      fin_flag = (t == (unsigned)M.nwin - 1u);
      if (fin_flag) chunk_ticket[chunk] = 0u;
    }
    __syncthreads();
    if (!fin_flag) return;
    __threadfence();
    for (int row = r0 + (int)threadIdx.x; row < r1; row += kWinThreads) {   // one thread per row, coalesced
      T tot = __ldcg(ypart + row);
      for (int ww = 1; ww < M.nwin; ++ww) tot += __ldcg(ypart + (size_t)ww * M.nrows + row);
      epi.row(row, tot, accS, accM);
    }
  }
  if constexpr (Epi::NS + Epi::NM > 0) {
    // finishing CTAs only: partials indexed by chunk => the fold order is run-independent
    reduce_and_finalize<T, Epi::NS, Epi::NM, Epi, kWinWarps>(accS, accM, rb, epi, chunk, nchunks);
  }
}

// ---------------------------------------------------------------------------
// Epilogues
// ---------------------------------------------------------------------------

// y = sum                                   (plain mul!)
template <typename T>
struct EpiStore {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* y;
  __device__ void row(int r, T s, T*, T*) const { y[r] = s; }
  __device__ void operator()(T*) const {}
};

// t = rho .* (A u)                          (kktsolver_indirect.jl:59-60)
template <typename T>
struct EpiScale {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* y;
  const T* rho;
  __device__ void row(int r, T s, T*, T*) const { y[r] = rho[r] * s; }
  __device__ void operator()(T*) const {}
};

// c = (A' t) + (P u) + sigma u ;  dot = u'c   (kktsolver_indirect.jl:61-65 + CG's dot(u, c))
// add_local = 0 on ranks > 0 of a row-sharded run: only rank 0 adds the replicated P/sigma terms.
template <typename T>
struct EpiKktOp {
  static constexpr int NS = 1, NM = 0;
  const int* done;
  T* c;
  const T* u;
  T sigma;
  const T* add;   // optional P u, computed by the P rows of the windowed kernel or by a separate launch (nullptr: the
                  // plain kernel traverses P's rows itself); read through L2, other CTAs of the same kernel may write it
  __device__ void row(int r, T s, T* accS, T*) const {
    const T ur = u[r];
    const T v = (add ? s + __ldcg(add + r) : s) + sigma * ur;
    c[r] = v;
    accS[0] += ur * v;
  }
  __device__ void operator()(T*) const {}
};

// rhs = x1 + A'(rho .* x2)                  (kktsolver_indirect.jl:52-54)
template <typename T>
struct EpiAddVec {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* y;
  const T* add;  // may be nullptr (ranks > 0)
  __device__ void row(int r, T s, T*, T*) const { y[r] = add ? s + add[r] : s; }
  __device__ void operator()(T*) const {}
};

// nu = rho .* (A y1 - x2)                   (kktsolver_indirect.jl:80-83), plugin entry
template <typename T>
struct EpiY2 {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* nu;
  const T* x2;
  const T* rho;
  __device__ void row(int r, T s, T*, T*) const { nu[r] = rho[r] * (s - x2[r]); }
  __device__ void operator()(T*) const {}
};

// y2 = A x1 - x2 ./ rho                    (kkt_mul!, kktsolver_indirect.jl:141-143)
template <typename T>
struct EpiKktFullLower {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  T* y;
  const T* x2;
  const T* rho;
  __device__ void row(int r, T s, T*, T*) const { y[r] = s - x2[r] / rho[r]; }
  __device__ void operator()(T*) const {}
};

// Fused ADMM tail on the last SpMV of the x-step:
//   nu   = rho .* (A y1 - x2)               (kktsolver_indirect.jl:80-83)
//   s_tl = 2 s - w_s - nu ./ rho            (solver.jl:55)
//   w_s  = w_s + alpha (s_tl - s)           (solver.jl:64)
//   tm   = rho .* (A y1)                    (optional: the warm-start product of the next CG solve, as EpiScale)
template <typename T>
struct EpiAdmmTail {
  static constexpr int NS = 0, NM = 0;
  const int* done;
  const T* x2;
  const T* rho;
  const T* s;
  const T* ws_in;
  T* ws_out;
  T alpha;
  T* tm;          // may be nullptr
  __device__ void row(int r, T sum, T*, T*) const {
    const T rh = rho[r];
    if (tm) tm[r] = rh * sum;
    const T nu = rh * (sum - x2[r]);
    const T sr = s[r], w = ws_in[r];
    const T s_tl = T(2) * sr - w - nu / rh;
    ws_out[r] = w + alpha * (s_tl - sr);
  }
  __device__ void operator()(T*) const {}
};

// Primal residual pass (residuals.jl:2-8,30-53,56-74):
//   max0 = |Einv (A x + s - b)|_inf, max1 = |Einv A x|_inf, max2 = |Einv s|_inf, max3 = |Einv b|_inf
template <typename T>
struct EpiPrimalRes {
  static constexpr int NS = 0, NM = 4;
  const int* done;
  const T* s;
  const T* b;
  const T* Einv;  // nullptr => identity
  T* ax_out;      // optional store of A x (nullptr = skip)
  __device__ void row(int r, T ax, T*, T* accM) const {
    const T e = Einv ? Einv[r] : T(1);
    const T sr = s[r], br = b[r];
    accM[0] = nanmax(accM[0], tabs(e * (ax + sr - br)));
    accM[1] = nanmax(accM[1], tabs(e * ax));
    accM[2] = nanmax(accM[2], tabs(e * sr));
    accM[3] = nanmax(accM[3], tabs(e * br));
    if (ax_out) ax_out[r] = ax;
  }
  __device__ void operator()(T*) const {}
};

// Dual residual pass over P rows with A'mu precomputed (residuals.jl:11-18,76-94,143-147):
//   max0 = |Dc (P x + q - A'mu)|_inf, max1 = |Dc P x|_inf, max2 = |Dc q|_inf, max3 = |Dc A'mu|_inf
//   sum0 = x'(P x), sum1 = q'x            with Dc = cinv * Dinv
template <typename T>
struct EpiDualRes {
  static constexpr int NS = 2, NM = 4;
  const int* done;
  const T* x;
  const T* q;
  const T* atmu;
  const T* Dinv;  // nullptr => identity
  T cinv;
  __device__ void row(int r, T px, T* accS, T* accM) const {
    const T d = (Dinv ? Dinv[r] : T(1)) * cinv;
    const T qr = q[r], ar = atmu[r], xr = x[r];
    accM[0] = nanmax(accM[0], tabs(d * (px + qr - ar)));
    accM[1] = nanmax(accM[1], tabs(d * px));
    accM[2] = nanmax(accM[2], tabs(d * qr));
    accM[3] = nanmax(accM[3], tabs(d * ar));
    accS[0] += xr * px;
    accS[1] += qr * xr;
  }
  __device__ void operator()(T*) const {}
};

// y = sum, max0 = |scale .* sum|_inf        (infeasibility.jl:12-18, 44-50)
template <typename T>
struct EpiStoreScaledMax {
  static constexpr int NS = 0, NM = 1;
  const int* done;
  T* y;              // may be nullptr
  const T* scale;    // nullptr => identity
  __device__ void row(int r, T s, T*, T* accM) const {
    if (y) y[r] = s;
    accM[0] = nanmax(accM[0], tabs((scale ? scale[r] : T(1)) * s));
  }
  __device__ void operator()(T*) const {}
};

}  // namespace cosmo
