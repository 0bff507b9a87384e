// win_pack.h -- the 9-byte entry of the packed fp64 column-windowed slabs (spmv_win_kernel, mat_update.cuh).
//
// A window is at most 25 600 doubles wide, so a window-local column needs 15 bits, and the values of one matrix span
// few binades.  A packed entry keeps the 52 mantissa bits and the sign of its value, a 4-bit exponent code and the
// column in 72 bits, split over two streams:
//   word  (8 B): [63] sign | [62:59] code | [58:52] column bits 0-6 | [51:0] mantissa
//   colhi (1 B): column bits 7-14
//   code 0      +-0 (the mantissa field is 0; slab padding is the all-zero word, +0.0)
//   code 1-14   biased exponent ebase + code - 1
//   code 15     escape: the value is esc[low 32 bits of the word], a per-matrix table of exact doubles (subnormals,
//               Inf, NaN with its payload, every exponent outside [ebase, ebase + 13])
// The decode is lossless: it returns the stored double bit for bit.  It touches only the high 32 bits of the word; the
// low word (mantissa bits 0-31, or the escape index) passes through.  The encoder runs on the device only: the slab
// kernels of mat_update.cuh call these functions when an engine is created and when its values are updated.  They
// are plain C++ with __host__ __device__ qualifiers, so a host program can check the very functions the kernels call.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define WP_HD __host__ __device__ __forceinline__
#else
#define WP_HD inline
#endif

namespace cosmo {
namespace winpack {

constexpr int kCodes = 14;            // binades of the exponent window
constexpr unsigned kEscape = 15u;
constexpr int kColBits = 15;
constexpr unsigned kMaxCol = (1u << kColBits) - 1u;
// a matrix keeps the 10 B layout when more than 1/kEscDen of its stored entries would be escapes
constexpr long long kEscDen = 256;

// (ebase - 1) << 20: added to code << 20 it gives the biased exponent field of the high word
WP_HD uint32_t exp_offset(int ebase) { return (uint32_t)(ebase - 1) << 20; }

// high word of the decoded double (meaningless for an escape)
WP_HD uint32_t decode_hi(uint32_t hi, uint32_t kexp) {
  const uint32_t t = hi & 0x78000000u;                        // code << 27
  return (hi & 0x800FFFFFu) | (t != 0u ? (t >> 7) + kexp : 0u);
}
WP_HD bool is_escape(uint32_t hi) { return (hi & 0x78000000u) == 0x78000000u; }
// window-local column from the high word and the column-high byte
WP_HD uint32_t decode_col(uint32_t hi, uint32_t colhi) { return ((hi >> 20) & 0x7Fu) | (colhi << 7); }

WP_HD uint64_t bits_of(double v) { uint64_t u; memcpy(&u, &v, 8); return u; }
WP_HD double double_of(uint64_t u) { double v; memcpy(&v, &u, 8); return v; }

// biased exponent of a finite normal value, 0 otherwise (zero, subnormal, Inf, NaN)
WP_HD int normal_exponent(double v) {
  const int e = (int)((bits_of(v) >> 52) & 0x7FF);
  return (e == 0 || e == 0x7FF) ? 0 : e;
}

// start of the kCodes-binade window that holds the most entries of a histogram of biased exponents (hist[1..2046])
inline int pick_ebase(const long long* hist) {
  int best = 1;
  long long best_cnt = -1, cnt = 0;
  for (int e = 1; e < 1 + kCodes; ++e) cnt += hist[e];
  for (int b = 1; b + kCodes - 1 <= 2046; ++b) {
    if (b > 1) cnt += hist[b + kCodes - 1] - hist[b - 1];
    if (cnt > best_cnt) { best_cnt = cnt; best = b; }
  }
  return best;
}

// exponent code of a value: 0 for +-0, 1-14 inside the window, kEscape otherwise
WP_HD unsigned code_of(double v, int ebase) {
  const uint64_t u = bits_of(v);
  if ((u << 1) == 0) return 0u;
  const int e = (int)((u >> 52) & 0x7FF);
  if (e == 0 || e == 0x7FF || e < ebase || e > ebase + kCodes - 1) return kEscape;
  return (unsigned)(e - ebase + 1);
}

// the packed word of (v, col); an escape stores esc_index in the low 32 bits, the caller stores v at esc[esc_index]
WP_HD uint64_t encode_word(double v, uint32_t col, int ebase, uint32_t esc_index) {
  const uint64_t u = bits_of(v);
  const unsigned code = code_of(v, ebase);
  const uint64_t mant = code == kEscape ? (uint64_t)esc_index : (u & 0x000FFFFFFFFFFFFFull);
  return (u & 0x8000000000000000ull) | ((uint64_t)code << 59) | ((uint64_t)(col & 0x7Fu) << 52) | mant;
}
WP_HD uint8_t encode_colhi(uint32_t col) { return (uint8_t)(col >> 7); }

// host reference of the device decode (same functions): the double and the column of one entry
inline double decode_value(uint64_t word, const double* esc, int ebase) {
  const uint32_t hi = (uint32_t)(word >> 32), lo = (uint32_t)word;
  if (is_escape(hi)) return esc[lo];
  return double_of(((uint64_t)decode_hi(hi, exp_offset(ebase)) << 32) | lo);
}

}  // namespace winpack
}  // namespace cosmo
