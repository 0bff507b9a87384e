// mat_update.cuh -- the values of P and A in the layouts the host built from their patterns: the one value path of
// engine creation and of cosmo_b200_update_matrices.
//
// The sparsity pattern fixes every layout: the CSR order of A and P, and the slot of every entry in the column-windowed
// slabs (win_fill_segment places entries by column only).  Maps say where each stored value comes from -- CSR position
// -> CSC index, slab column position -> CSC index or -1 for padding -- and the CSC values are gathered through them.
// The 9 B slabs are encoded with the win_pack.h functions: one exponent histogram, the window base picked on the host,
// escapes counted per (window, row) segment and numbered in slab order, so the words, the escape table and the layout
// decision depend on the pattern and the values alone.
// Included from engine.cu (after common.cuh).
#pragma once
#include "win_pack.h"

namespace cosmo {
namespace matup {

// out[i] = v[src[i]]
template <typename T>
__global__ void __launch_bounds__(kBlock) gather_kernel(long long n, const int* __restrict__ src, const T* __restrict__ v,
                                                        T* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = v[src[i]];
}

// histogram of the biased exponents of the finite normal values (the exponent window, pick_ebase); integer atomics, so the
// counts do not depend on the schedule
__global__ void __launch_bounds__(kBlock) exp_hist_kernel(long long n, const double* __restrict__ v,
                                                          unsigned long long* __restrict__ hist) {
  __shared__ unsigned int h[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) h[i] = 0u;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(&h[winpack::normal_exponent(v[i])], 1u);
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += blockDim.x)
    if (h[i]) atomicAdd(&hist[i], (unsigned long long)h[i]);
}

// value position of the entry at column position `idx` of a segment of `kpad` entries starting at `s`: the
// instruction-coalesced value order spmv_win_kernel loads (load8_coalesced: EPL values per 16-byte load)
template <int EPL>
__device__ __forceinline__ long long value_pos(long long s, int kpad, int idx) {
  const int st = idx >> 8, l = (idx & 255) >> 3, i = idx & 7;
  const int ls = min(32, (kpad >> 3) - 32 * st);
  return s + (long long)st * 256 + (long long)(i / EPL) * (EPL * ls) + (long long)l * EPL + (i % EPL);
}

// f(g, s, kpad, lane) for every (window, row) segment g = w * nr + r of a slab, one warp per segment
template <typename F>
__device__ __forceinline__ void for_each_segment(int nwin, int nr, const int* __restrict__ rp, F&& f) {
  const int lane = threadIdx.x & 31;
  const long long nseg = (long long)nwin * nr, warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; g < nseg; g += warps) {
    const int w = (int)(g / nr), r = (int)(g % nr);
    const int s = rp[(size_t)w * (nr + 1) + r];
    f(g, s, rp[(size_t)w * (nr + 1) + r + 1] - s, lane);
  }
}

// 10 B / 6 B slab values: w_val at the value position of every column position, zero on padding
template <typename T>
__global__ void __launch_bounds__(kBlock) slab_gather_kernel(int nwin, int nr, const int* __restrict__ rp,
                                                             const int* __restrict__ wsrc, const T* __restrict__ v,
                                                             T* __restrict__ w_val) {
  for_each_segment(nwin, nr, rp, [&](long long, int s, int kpad, int lane) {
    for (int idx = lane; idx < kpad; idx += 32) {
      const int k = wsrc[s + idx];
      w_val[value_pos<16 / (int)sizeof(T)>(s, kpad, idx)] = k >= 0 ? v[k] : T(0);
    }
  });
}

// escapes of every segment under the window base `ebase` (padding is +0.0, code 0)
__global__ void __launch_bounds__(kBlock) slab_esc_count_kernel(int nwin, int nr, const int* __restrict__ rp,
                                                                const int* __restrict__ wsrc, const double* __restrict__ v,
                                                                int ebase, int* __restrict__ cnt) {
  for_each_segment(nwin, nr, rp, [&](long long g, int s, int kpad, int lane) {
    int c = 0;
    for (int idx = lane; idx < kpad; idx += 32) {
      const int k = wsrc[s + idx];
      c += k >= 0 && winpack::code_of(v[k], ebase) == winpack::kEscape;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) cnt[g] = c;
  });
}

// 9 B words, column-high bytes and escape table of a slab (win_pack.h): escapes take consecutive slots from the segment's
// offset in column-position order.  The window-local column comes from w_col (FROM_COL: the slab was 10 B) or is
// decoded from the word and colhi the slab already holds (the column bits never change).
template <bool FROM_COL>
__global__ void __launch_bounds__(kBlock) slab_encode_kernel(int nwin, int nr, const int* __restrict__ rp,
                                                             const int* __restrict__ wsrc, const double* __restrict__ v,
                                                             int ebase, const long long* __restrict__ esc_off,
                                                             const unsigned short* __restrict__ w_col,
                                                             unsigned long long* __restrict__ word,
                                                             unsigned char* __restrict__ colhi, double* __restrict__ esc) {
  namespace wp = winpack;
  for_each_segment(nwin, nr, rp, [&](long long g, int s, int kpad, int lane) {
    long long ei = esc_off[g];
    for (int base = 0; base < kpad; base += 32) {   // kpad is warp-uniform: every lane takes part in the ballot
      const int idx = base + lane;
      const bool act = idx < kpad;
      double x = 0.0;
      uint32_t col = 0;
      long long pv = 0;
      if (act) {
        const int k = wsrc[s + idx];
        x = k >= 0 ? v[k] : 0.0;
        pv = value_pos<2>(s, kpad, idx);
        if (FROM_COL) {
          col = w_col[s + idx];
          colhi[s + idx] = wp::encode_colhi(col);
        } else {
          col = wp::decode_col((uint32_t)(word[pv] >> 32), colhi[s + idx]);
        }
      }
      const bool e = act && wp::code_of(x, ebase) == wp::kEscape;
      const unsigned bal = __ballot_sync(0xffffffffu, e);
      uint32_t slot = 0;
      if (e) {
        slot = (uint32_t)(ei + __popc(bal & ((1u << lane) - 1u)));
        esc[slot] = x;
      }
      if (act) word[pv] = wp::encode_word(x, col, ebase, slot);
      ei += __popc(bal);
    }
  });
}

// the window-local columns of a 9 B slab, for its conversion to the 10 B layout
__global__ void __launch_bounds__(kBlock) slab_unpack_col_kernel(int nwin, int nr, const int* __restrict__ rp,
                                                                 const unsigned long long* __restrict__ word,
                                                                 const unsigned char* __restrict__ colhi,
                                                                 unsigned short* __restrict__ w_col) {
  for_each_segment(nwin, nr, rp, [&](long long, int s, int kpad, int lane) {
    for (int idx = lane; idx < kpad; idx += 32)
      w_col[s + idx] = (unsigned short)winpack::decode_col((uint32_t)(word[value_pos<2>(s, kpad, idx)] >> 32), colhi[s + idx]);
  });
}

}  // namespace matup
}  // namespace cosmo
