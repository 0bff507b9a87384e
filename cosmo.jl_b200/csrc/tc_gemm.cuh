// tc_gemm.cuh -- fp64-accurate products of symmetric matrices on the Hopper tensor cores (sm_90a).
//
// The PSD projection of a large cone (convexset.jl:219-263 in the reference: dsyevr + clamp + syrk) is computed here
// as  Pi_+(X) = (X + sign(X) X) / 2  with sign(X) from a Newton-Schulz iteration (psd_tc.cuh) -- nothing but
// N x N x N products of symmetric, commuting matrices.  The data-sheet int8 rate of the H100 SXM tensor cores is 30x
// their fp64 rate (1979 vs 67 TOP/s), so every product is evaluated by error-free slicing (Ozaki scheme I):
//
//     M[r, :] = 2^(e_r - 6) * sum_p D_p[r, :] * 128^-(p-1),   D_p int8 digits in [-64, 64]   (slice_rows_kernel)
//     (A B)[m, n] = sA[m] sB[n] * sum_s 128^-(s-2) G_s[m, n],  G_s = sum_{p+q=s} A_p B_q^T     (int32, EXACT)
//
// G_s is accumulated by wgmma.mma_async s32.s8.s8 in registers (|G_s| <= 8 * K * 64^2 < 2^31 for K <= 65536), the sum
// over s runs in fp64 registers of the same threads (acc += 128^-(s-2) G_s, least significant groups first), so the
// only rounding errors are the truncation of the slices (2^-7k relative to the row maximum) and one fp64 rounding per
// group.
//
// Kernel anatomy (one persistent CTA per SM, three warpgroups):
//   warpgroup 0   TMA producer: one warp issues cp.async.bulk.tensor.2d, 128-row x 128-byte boxes (= the tiles of 4
//                 slices for one K step of 32, see the layout note below), 128-byte hardware swizzle, into a ring of
//                 six 32 KB units {A box, B box}, mbarrier complete_tx
//   warpgroups 1, 2   consumers: warpgroup c owns rows [64 c, 64 c + 64) of the 128 x 128 output tile.  Per group s
//                 it issues wgmma.m64n128k32 (A and B from shared-memory descriptors) for every slice pair p + q = s of
//                 each K step into one 64-register int32 accumulator, releases the ring unit, and after the last K
//                 step folds the exact int32 sums into its 64 fp64 accumulators.  The final epilogue fuses
//                 out = c0 * (A B) + c1 * D + c2 * I, the mirrored store (the product of commuting symmetric matrices
//                 is symmetric: only tiles of the upper triangle are computed) and two Frobenius reductions.
// One int32 accumulator per group is what the register file affords next to the 64 fp64 accumulators of a thread
// (64 + 128 of the 232 registers a consumer thread gets), so each group streams its operand boxes once per tile.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>

#include "host.cuh"

namespace cosmo {
namespace tc {

constexpr int kTile = 128;         // output tile side = rows of one operand box = wgmma N = 2 x wgmma M
constexpr int kSlices = 8;         // slices stored per matrix (unused ones are zero)
constexpr int kKStep = 32;         // K per stage = K of one wgmma.m64n128k32.s8
constexpr int kBoxBytes = kTile * 128;   // one TMA box: 128 rows x (4 slices x 32 K-bytes), 128-byte swizzle
constexpr int kUnitBytes = 2 * kBoxBytes;    // ring unit: {A box, B box} of slices 0-3 (or of slices 4-7)
constexpr int kUnits = 6;                    // 192 KB ring: 3 K steps in flight when a group needs both halves, 6 otherwise
constexpr int kThreads = 384;      // warpgroup 0: TMA (warp 0 issues, 1-3 idle); warpgroups 1, 2: wgmma + epilogue
constexpr int kEpiWarps = 8;

// Layout of a sliced operand: int8 [row][K / 32][slice 0..7][32], i.e. a row of Np * 8 bytes in which the 8 slices of
// the same 32 K-values are adjacent.  One 128-byte TMA row therefore carries 4 slices of one K step, a 128 x 128-byte
// box is the operand tile of 4 slices at once, and the tile of slice j inside the box is addressed like the j-th
// K sub-step of an ordinary 128-byte-swizzled K-major tile (descriptor start address + 32 j bytes).
//
// With K slices and G groups the groups s = p + q run from G + 1 down to 2; group s pairs the A slices
// p = group_p_lo .. group_p_hi with the B slices q = s - p.
// G >= K is the number of groups kept: G = K is the classical truncation (error ~ K 2^-7K relative to the row maxima),
// every further group gains 7 bits; G = K + 2 leaves only the truncation of the operands themselves (2^-7K per
// element): with K = 8 the product is then more accurate than dgemm.
__host__ __device__ constexpr int group_p_lo(int k, int s) { return s - k > 1 ? s - k : 1; }
__host__ __device__ constexpr int group_p_hi(int k, int s) { return s - 1 < k ? s - 1 : k; }
// a group needs the slices 4-7 of either operand <=> it occupies two ring units per K step (kUnits is even and the
// number of K steps is even, so a two-unit step never wraps inside).  The slices 0-3 are needed by every group
// (G <= K + 2 keeps group_p_lo <= 3).
__host__ __device__ constexpr int group_units(int k, int s) { return (group_p_hi(k, s) > 4 || s - group_p_lo(k, s) > 4) ? 2 : 1; }
__host__ __device__ constexpr int total_products(int k, int g) {
  int n = 0;
  for (int s = 2; s <= g + 1; ++s) n += group_p_hi(k, s) - group_p_lo(k, s) + 1;
  return n;
}

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra LAB_DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "LAB_DONE:\n\t}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P1;\n\telect.sync _|P1, 0xffffffff;\n\tselp.b32 %0, 1, 0, P1;\n\t}\n" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// d += A[smem] * B[smem]^T on the 64 x 128 block of the calling warpgroup, int8 x int8 -> int32, K = 32.
// d[4 j + i] of lane l in warp w of the warpgroup is element (16 w + l / 4 + 8 (i / 2), 8 j + 2 (l % 4) + i % 2).
__device__ __forceinline__ void wgmma_i8(int32_t (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
        "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
        "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
        "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]),
        "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
        "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
        "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]),
        "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc)
      : "memory");
}
// shared-memory matrix descriptor of a K-major operand tile inside a 128-row x 128-byte box written by TMA with the
// 128-byte swizzle (atoms of 8 rows x 128 bytes: stride between atoms along M / N = 1024 bytes, the leading byte offset
// is unused by swizzled K-major layouts); `saddr16` is the shared-memory byte address >> 4 of the first row
// + 32 * (slice within the box)
constexpr uint64_t kDescHi = (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);   // LBO 1, SBO, SWIZZLE_128B
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr16) { return kDescHi | (uint64_t)(saddr16 & 0x3FFFu); }

// (double)v for an int32 v without the conversion unit: 2^52 + 2^31 + v is exactly representable, its bit pattern is
// {0x43300000, v ^ 0x80000000}
__device__ __forceinline__ double biased_double(uint32_t v) { return __hiloint2double(0x43300000, (int)(v ^ 0x80000000u)); }
constexpr double kBias = 4503599627370496.0 + 2147483648.0;

// ---------------------------------------------------------------------------------------------------------------
// Slicing: one CTA per row.  scale[r] = 2^(e_r - 6) with 2^e_r > max |M[r, :]|, so t = x / scale is in (-64, 64).
// The K digits are the balanced base-128 digits of the fixed-point number v = rn(t 2^(7K-7)) (unit of the last kept
// digit = 1): with the bias B = 64 sum_{j<K} 128^j added, u = v + B >= 0 and the 7-bit FIELDS of u are digit + 64 --
// no carries, no per-digit rounding: one fp64 multiply and one conversion per element, integer field extraction per
// digit (the first version took rint / subtract / scale / convert per digit in fp64).  Digits are in [-64, 63], the
// leading one in [-64, 64]; all of it exact.  Output layout: see the note above.
// ---------------------------------------------------------------------------------------------------------------
template <int K>
struct SliceFix {
  static constexpr int kShift = 7 * K - 7;
  __host__ __device__ static constexpr unsigned long long bias() {
    unsigned long long b = 0;
    for (int j = 0; j < K; ++j) b += 64ull << (7 * j);
    return b;
  }
};

template <int K>
__host__ __device__ __forceinline__ unsigned long long slice_fixed(double t) {
  const double s = t * (double)(1ull << SliceFix<K>::kShift);
#ifdef __CUDA_ARCH__
  const long long v = __double2ll_rn(s);
#else
  const long long v = llrint(s);
#endif
  return (unsigned long long)(v + (long long)SliceFix<K>::bias());
}

// digit p (0 = most significant) of u[0..3] as the four int8 bytes of one word
template <int K>
__host__ __device__ __forceinline__ uint32_t slice_pack4(const unsigned long long* u, int p) {
  const int off = 7 * (K - 1 - p);
  uint32_t w = 0;
  if (p == 0) {   // the leading field runs over [0, 128]
#pragma unroll
    for (int j = 0; j < 4; ++j) w |= ((uint32_t)((int)(u[j] >> off) - 64) & 0xffu) << (8 * j);
    return w;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) w |= ((uint32_t)(u[j] >> off) & 127u) << (8 * j);
  // field f -> int8(f - 64), four bytes at a time: f >= 64: f ^ 0x40;  f < 64: (f ^ 0x40) | 0x80 = f + 192
  const uint32_t x = w ^ 0x40404040u;
  return x | ((x & 0x40404040u) << 1);
}

// The row is read once, coalesced, for the maximum and parked in shared memory (element c at c + c / 8: the padding
// makes the 8-consecutive-columns-per-thread reads of the second pass conflict-free; read straight from global memory
// they cost 16 L1 wavefronts per load instruction).  Rows too long for shared memory (`staged` = 0) are re-read.
constexpr int kSliceStageMaxBytes = 200 * 1024;
__host__ __device__ constexpr size_t slice_stage_bytes(int N) { return ((size_t)N + (size_t)N / 8 + 8) * sizeof(double); }

template <typename T, int K>
__global__ void __launch_bounds__(256) slice_rows_kernel(const T* __restrict__ M, int N, int Np, int8_t* __restrict__ slices,
                                                        double* __restrict__ scale, int staged) {
  extern __shared__ __align__(16) double slice_srow[];
  const int r = blockIdx.x;
  const T* row = M + (size_t)r * N;   // symmetric: row r == column r of the column-major matrix
  __shared__ double red[8];
  double mx = 0.0;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    const double v = (double)row[c];
    if (staged) slice_srow[c + (c >> 3)] = v;
    mx = fmax(mx, fabs(v));
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < 8; ++w) mx = fmax(mx, red[w]);
  int e = 0;
  if (mx > 0.0 && mx <= 1.7976931348623157e308) frexp(mx, &e);   // mx = f 2^e, f in [0.5, 1)  =>  |x| < 2^e
  // Contract: every row whose maximum is a normal number is sliced exactly as at scale 1 (same digits, scale[r] a power
  // of two).  scale[r] = 2^(e - 6) is subnormal for e < -1016 but still exact (powers of two down to 2^-1074 are), and the
  // epilogue forms acc * sA * sB left to right, so the product keeps its accuracy relative to |A| |B|.  Rows whose maximum
  // is itself subnormal are sliced as if it were 2^-1022 (e = -1021): their digits have fewer significant bits, i.e. they
  // are exact to 2^-7K * 2^-1021 in absolute terms, not relative to the row maximum.
  e = e < -1021 ? -1021 : e;
  if (threadIdx.x == 0) scale[r] = ldexp(1.0, e - 6);
  // 2^(6 - e) as two factors: over the whole normal range each factor is a normal number, and x * inv0 * inv1 is the
  // exact power-of-two scaling (2^(6 - e) alone overflows for e < -1017)
  const double inv0 = ldexp(1.0, (6 - e) / 2), inv1 = ldexp(1.0, (6 - e) - (6 - e) / 2);
  int8_t* out_row = slices + (size_t)r * Np * kSlices;
  for (int c0 = threadIdx.x * 8; c0 < N; c0 += blockDim.x * 8) {
    unsigned long long u[8];
    const double* sp = slice_srow + c0 + (c0 >> 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      double x = 0.0;
      if (c0 + j < N) x = staged ? sp[j] : (double)row[c0 + j];
      u[j] = slice_fixed<K>(x * inv0 * inv1);
    }
    int8_t* dst = out_row + (size_t)(c0 >> 5) * (kSlices * 32) + (c0 & 31);
#pragma unroll
    for (int p = 0; p < K; ++p)
      *reinterpret_cast<uint2*>(dst + p * 32) = make_uint2(slice_pack4<K>(u, p), slice_pack4<K>(u + 4, p));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The product kernel
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
struct GemmArgs {
  int N, Np, ntiles, store;          // store: 1 = write `out`
  const int2* tiles;                 // (bi, bj), bi <= bj: tiles of the upper triangle
  const double* scaleA;              // Np row scales of the A operand
  const double* scaleB;              // Np row (= column) scales of the B operand
  T* out;                            // N x N, ld = N (symmetric, mirrored store)
  const T* D;                        // optional: out = c0 * (A B) + c1 * D + c2 * I
  const T* E;                        // optional reference of the second reduction
  int e_identity;                    // 1: second reduction against the identity
  const double* coef;                // device scalars c0, c1, c2
  double* partial;                   // 2 per tile: sum w out^2, sum w (E - out)^2   (w: 1 on the diagonal, 2 above it)
};

struct PipeState { int unit; uint32_t phase; };   // position in the ring of kUnits units

__device__ __forceinline__ void pipe_advance(PipeState& st, int n) {
  st.unit += n;
  if (st.unit == kUnits) { st.unit = 0; st.phase ^= 1; }
}

template <typename T, int K, int G>
__global__ void __launch_bounds__(kThreads, 1) ozaki_gemm_kernel(const __grid_constant__ CUtensorMap tmapA,
                                                                 const __grid_constant__ CUtensorMap tmapB, const GemmArgs<T> args) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[kUnits], empty_bar[kUnits];
  __shared__ double red[kEpiWarps][2];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kUnits; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }   // 2: one per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nk = args.Np / kKStep;

  // register re-distribution (setmaxnreg is per warpgroup): the producer needs few registers, a consumer thread holds
  // 64 int32 wgmma accumulators and 64 fp64 sums
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      // ===== TMA producer (warp-uniform loop, one elected lane issues) =====
      PipeState st{0, 0};
      for (int t = blockIdx.x; t < args.ntiles; t += gridDim.x) {
        const int2 tl = args.tiles[t];
        const int m0 = tl.x * kTile, n0 = tl.y * kTile;
        for (int s = G + 1; s >= 2; --s) {
          const int nu = group_units(K, s);
          for (int ks = 0; ks < nk; ++ks) {
            for (int h = 0; h < nu; ++h) {
              mbar_wait(&empty_bar[st.unit], st.phase ^ 1);
              if (elect_one()) {
                mbar_expect_tx(&full_bar[st.unit], (uint32_t)kUnitBytes);
                const uint32_t dst = smem_u32(smem) + (uint32_t)st.unit * kUnitBytes;
                const int c0 = ks * (kSlices * 32) + h * 128;
                tma_load_2d(dst, &tmapA, &full_bar[st.unit], c0, m0);
                tma_load_2d(dst + kBoxBytes, &tmapB, &full_bar[st.unit], c0, n0);
              }
              __syncwarp();
              pipe_advance(st, 1);
            }
          }
        }
      }
    }
  } else {
    // ===== consumers: wgmma + epilogue =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1;       // rows [64 wg, 64 wg + 64) of the tile
    const int ew = warp - 4;
    const int wq = warp & 3;              // rows [16 wq, 16 wq + 16) of the warpgroup's block
    const uint32_t a_row16 = (uint32_t)(wg * 64 * 128) >> 4;   // 64 rows of 128 bytes: whole swizzle atoms
    const double c0 = args.coef[0], c1 = args.coef[1], c2 = args.coef[2];
    PipeState st{0, 0};
    for (int t = blockIdx.x; t < args.ntiles; t += gridDim.x) {
      const int2 tl = args.tiles[t];
      double acc[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.0;
      for (int s = G + 1; s >= 2; --s) {
        const int plo = group_p_lo(K, s), phi = group_p_hi(K, s), nu = group_units(K, s);
        int32_t d[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) d[j] = 0;
        for (int ks = 0; ks < nk; ++ks) {
          mbar_wait(&full_bar[st.unit], st.phase);
          if (nu == 2) mbar_wait(&full_bar[st.unit + 1], st.phase);
          const uint32_t sbase16 = (smem_u32(smem) + (uint32_t)st.unit * kUnitBytes) >> 4;
          wgmma_fence();
          for (int p = plo; p <= phi; ++p) {
            const int q = s - p;
            const uint32_t a_off = (uint32_t)((((p - 1) / 4) * kUnitBytes + ((p - 1) % 4) * 32) >> 4) + a_row16;
            const uint32_t b_off = (uint32_t)((((q - 1) / 4) * kUnitBytes + kBoxBytes + ((q - 1) % 4) * 32) >> 4);
            wgmma_i8(d, smem_desc(sbase16 + a_off), smem_desc(sbase16 + b_off));
          }
          wgmma_commit();
          wgmma_wait_all();
          if ((threadIdx.x & 127) == 0) {
            mbar_arrive(&empty_bar[st.unit]);
            if (nu == 2) mbar_arrive(&empty_bar[st.unit + 1]);
          }
          pipe_advance(st, nu);
        }
        // acc += 128^-(s-2) G_s, exactly converted
        const double sc = ldexp(1.0, -7 * (s - 2));
        const double nb = -kBias * sc;
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] += fma(biased_double((uint32_t)d[j]), sc, nb);   // fma is exact: v * sc
      }
      // ---- final epilogue of the tile ----
      double r0 = 0.0, r1 = 0.0;
      const int N = args.N;
      const int gm0 = tl.x * kTile + wg * 64 + wq * 16 + (lane >> 2);
      const int gn0 = tl.y * kTile + 2 * (lane & 3);
      const double sa0 = gm0 < N ? args.scaleA[gm0] : 0.0, sa1 = gm0 + 8 < N ? args.scaleA[gm0 + 8] : 0.0;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int gm = gm0 + 8 * ((j >> 1) & 1);
        const int gn = gn0 + 8 * (j >> 2) + (j & 1);
        if (gm >= N || gn >= N || gm > gn) continue;      // upper triangle only; the mirror is written below
        double o = c0 * (acc[j] * (((j >> 1) & 1) ? sa1 : sa0) * args.scaleB[gn]);
        const size_t tidx = (size_t)gn * N + gm;        // element (gm, gn) of a column-major matrix
        if (args.D) o += c1 * (double)args.D[tidx];
        if (gm == gn) o += c2;
        const double w = (gm == gn) ? 1.0 : 2.0;
        r0 += w * o * o;
        if (args.e_identity || args.E) {
          const double ref = args.E ? (double)args.E[tidx] : ((gm == gn) ? 1.0 : 0.0);
          r1 += w * (ref - o) * (ref - o);
        }
        if (args.store) {
          args.out[tidx] = (T)o;
          if (gm != gn) args.out[(size_t)gm * N + gn] = (T)o;
        }
      }
      if (args.partial) {
        for (int o = 16; o > 0; o >>= 1) {
          r0 += __shfl_xor_sync(0xffffffffu, r0, o);
          r1 += __shfl_xor_sync(0xffffffffu, r1, o);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");     // previous tile's reader is done with red[]
        if (lane == 0) { red[ew][0] = r0; red[ew][1] = r1; }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ew == 0 && lane == 0) {
          double a = 0.0, b = 0.0;
          for (int w = 0; w < kEpiWarps; ++w) { a += red[w][0]; b += red[w][1]; }
          args.partial[2 * t] = a;
          args.partial[2 * t + 1] = b;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// One sliced operand: int8 [Np][Np / 32][8][32] + Np scales, and its tensor map for the current Np.
struct Sliced {
  DevBuf<int8_t> d;
  DevBuf<double> scale;
  CUtensorMap map;
  int capNp = 0, mapNp = 0;
  void ensure(int Np) {
    if (Np <= capNp) return;
    capNp = 0; mapNp = 0;
    d.alloc((size_t)kSlices * Np * Np, false);
    scale.alloc(Np, false);
    capNp = Np;
  }
  // zero padding rows / columns and unused slices: called when the shape of the cone changes
  void clear(int Np, cudaStream_t st) {
    mapNp = 0;
    CUDA_TRY(cudaMemsetAsync(d.p, 0, (size_t)kSlices * Np * Np, st));
    CUDA_TRY(cudaMemsetAsync(scale.p, 0, (size_t)Np * sizeof(double), st));
  }
  void make_map(int Np) {
    if (mapNp == Np) return;
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) throw EngineError{COSMO_B200_ERR_CUDA, "cuTensorMapEncodeTiled is not available"};
    const cuuint64_t dims[2] = {(cuuint64_t)Np * kSlices, (cuuint64_t)Np};
    const cuuint64_t strides[1] = {(cuuint64_t)Np * kSlices};
    const cuuint32_t box[2] = {128, (cuuint32_t)kTile};
    const cuuint32_t estr[2] = {1, 1};
    if (enc(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d.p, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      throw EngineError{COSMO_B200_ERR_CUDA, "cuTensorMapEncodeTiled failed"};
    mapNp = Np;
  }
};

template <typename T>
struct OzakiGemm {
  DevBuf<int2> tiles_d;
  int tilesNp = 0, ntiles = 0;
  int k = 8, g = 10, num_sms = 132;
  int N = 0, Np = 0;

  static constexpr int smem_bytes() { return kUnits * kUnitBytes + 1024; }
  // supported (slices, groups): (8, 10) exact-fp64 default, (8, 8) and (7, 7) classical truncations, (6, 8) and (4, 6)
  // for the fp32 model type
  template <int K, int G>
  static void set_attr() {
    CUDA_TRY(cudaFuncSetAttribute(ozaki_gemm_kernel<T, K, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes()));
  }
  template <int K>
  static void set_slice_attr() {
    CUDA_TRY(cudaFuncSetAttribute(slice_rows_kernel<T, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSliceStageMaxBytes));
  }
  static bool supported(int k_, int g_) {
    return (k_ == 8 && (g_ == 10 || g_ == 8)) || (k_ == 7 && g_ == 7) || (k_ == 6 && g_ == 8) || (k_ == 4 && g_ == 6);
  }
  void configure(int k_, int g_) {
    if (!supported(k_, g_)) throw EngineError{COSMO_B200_ERR_INVALID, "tc::OzakiGemm: unsupported (slices, groups)"};
    k = k_; g = g_;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    // per device, every time: function attributes are per device and cheap to set
    set_attr<8, 10>(); set_attr<8, 8>(); set_attr<7, 7>(); set_attr<6, 8>(); set_attr<4, 6>();
    set_slice_attr<8>(); set_slice_attr<7>(); set_slice_attr<6>(); set_slice_attr<4>();
  }
  void set_shape(int N_, cudaStream_t st) {
    N = N_;
    Np = (N + kTile - 1) / kTile * kTile;
    if (tilesNp != Np) {
      const int nt = Np / kTile;
      std::vector<int2> tl;
      for (int bj = 0; bj < nt; ++bj)
        for (int bi = 0; bi <= bj; ++bi) tl.push_back(make_int2(bi, bj));
      tilesNp = 0;
      tiles_d.alloc(tl.size(), false);
      tiles_d.upload(tl.data(), tl.size(), st);
      CUDA_TRY(cudaStreamSynchronize(st));
      ntiles = (int)tl.size();
      tilesNp = Np;
    }
  }
  // slices of an N x N symmetric matrix (ld = N) into `sl` (padding rows / columns must have been cleared)
  void slice(const T* M, Sliced& sl, cudaStream_t st) {
    const int staged = slice_stage_bytes(N) <= (size_t)kSliceStageMaxBytes ? 1 : 0;
    const size_t sm = staged ? slice_stage_bytes(N) : 0;
    if (k == 8) slice_rows_kernel<T, 8><<<N, 256, sm, st>>>(M, N, Np, sl.d.p, sl.scale.p, staged);
    else if (k == 7) slice_rows_kernel<T, 7><<<N, 256, sm, st>>>(M, N, Np, sl.d.p, sl.scale.p, staged);
    else if (k == 6) slice_rows_kernel<T, 6><<<N, 256, sm, st>>>(M, N, Np, sl.d.p, sl.scale.p, staged);
    else slice_rows_kernel<T, 4><<<N, 256, sm, st>>>(M, N, Np, sl.d.p, sl.scale.p, staged);
    CUDA_TRY(cudaGetLastError());
  }
  // out = c0 (A B) + c1 D + c2 I   (+ reductions into partial[2 * ntiles])
  void gemm(Sliced& A, Sliced& B, T* out, const T* D, const T* E, int e_identity, const double* coef_d, double* partial,
            cudaStream_t st) {
    A.make_map(Np);
    B.make_map(Np);
    GemmArgs<T> a;
    a.N = N; a.Np = Np; a.ntiles = ntiles; a.store = out ? 1 : 0;
    a.tiles = tiles_d.p; a.scaleA = A.scale.p; a.scaleB = B.scale.p; a.out = out; a.D = D; a.E = E; a.e_identity = e_identity;
    a.coef = coef_d; a.partial = partial;
    const int grid = std::min(ntiles, num_sms);
    if (k == 8 && g == 10) ozaki_gemm_kernel<T, 8, 10><<<grid, kThreads, smem_bytes(), st>>>(A.map, B.map, a);
    else if (k == 8) ozaki_gemm_kernel<T, 8, 8><<<grid, kThreads, smem_bytes(), st>>>(A.map, B.map, a);
    else if (k == 7) ozaki_gemm_kernel<T, 7, 7><<<grid, kThreads, smem_bytes(), st>>>(A.map, B.map, a);
    else if (k == 6) ozaki_gemm_kernel<T, 6, 8><<<grid, kThreads, smem_bytes(), st>>>(A.map, B.map, a);
    else ozaki_gemm_kernel<T, 4, 6><<<grid, kThreads, smem_bytes(), st>>>(A.map, B.map, a);
    CUDA_TRY(cudaGetLastError());
  }
};

}  // namespace tc
}  // namespace cosmo
