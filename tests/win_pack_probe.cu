// Host-side round trip of the packed fp64 slab entry (csrc/win_pack.h): encode_word / encode_colhi and the
// __host__ __device__ decode_hi / is_escape / decode_col that spmv_win_kernel calls, on the host, without a GPU
// (compiled by tests/test_win_pack_cpu.py with nvcc; nothing is launched).  Every decoded double must be the encoded
// one bit for bit, and every column the encoded column.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "win_pack.h"

using namespace cosmo::winpack;

static unsigned long long rng_state = 0x9E3779B97F4A7C15ull;
static unsigned long long next_u64() {   // xorshift64
  rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
  return rng_state;
}

static long long n_checked = 0, bad = 0;

// encode (v, col) against the window starting at ebase, decode it the way the kernel does, compare bits
static void round_trip(double v, unsigned col, int ebase, std::vector<double>& esc) {
  const unsigned code = code_of(v, ebase);
  const unsigned slot = (unsigned)esc.size();
  if (code == kEscape) esc.push_back(v);
  const uint64_t word = encode_word(v, col, ebase, slot);
  const uint8_t hb = encode_colhi(col);
  const uint32_t hi = (uint32_t)(word >> 32), lo = (uint32_t)word;
  double d;
  if (is_escape(hi)) d = esc[lo];
  else d = double_of(((uint64_t)decode_hi(hi, exp_offset(ebase)) << 32) | lo);
  const bool ok = bits_of(d) == bits_of(v) && decode_col(hi, hb) == col && is_escape(hi) == (code == kEscape) &&
                  bits_of(decode_value(word, esc.data(), ebase)) == bits_of(v);
  if (!ok) {
    if (bad < 10)
      printf("mismatch: v=%a (%016llx) col=%u ebase=%d code=%u -> %a (%016llx) col %u\n", v,
             (unsigned long long)bits_of(v), col, ebase, code, d, (unsigned long long)bits_of(d), decode_col(hi, hb));
    ++bad;
  }
  ++n_checked;
}

static void expect(bool c, const char* what) {
  if (!c) { printf("failed: %s\n", what); ++bad; }
}

int main() {
  const unsigned cols[] = {0u, 1u, 127u, 128u, 255u, 256u, 16383u, 16384u, 25599u, 32767u};
  std::vector<double> esc;
  esc.reserve(1 << 22);
  // random bit patterns: every exponent field (zero, subnormal, normal, Inf, NaN) and both signs, against windows at
  // both ends of the exponent range and in between
  const int bases[] = {1, 2, 500, 1000, 1013, 1023, 1500, 2032, 2033};
  for (int ebase : bases) {
    for (int it = 0; it < 400000; ++it) {
      uint64_t u = next_u64();
      if (it & 1) {   // half of them inside or next to the window
        const int e = ebase - 1 + (int)(next_u64() % (kCodes + 2));
        u = (u & 0x800FFFFFFFFFFFFFull) | ((uint64_t)(e & 0x7FF) << 52);
      }
      round_trip(double_of(u), (unsigned)(next_u64() % (kMaxCol + 1)), ebase, esc);
    }
    esc.clear();
  }
  // specials: +-0, subnormals, +-Inf, NaNs with payloads, the largest finite values
  const uint64_t specials[] = {0x0000000000000000ull, 0x8000000000000000ull, 0x0000000000000001ull, 0x8000000000000001ull,
                               0x000FFFFFFFFFFFFFull, 0x800FFFFFFFFFFFFFull, 0x0008000000000000ull, 0x7FF0000000000000ull,
                               0xFFF0000000000000ull, 0x7FF8000000000000ull, 0xFFF8000000000000ull, 0x7FF0000000000001ull,
                               0x7FF4000000ABCDEFull, 0xFFFFFFFFFFFFFFFFull, 0x7FEFFFFFFFFFFFFFull, 0xFFEFFFFFFFFFFFFFull,
                               0x0010000000000000ull, 0x8010000000000000ull};
  for (int ebase : bases)
    for (uint64_t u : specials)
      for (unsigned c : cols) round_trip(double_of(u), c, ebase, esc);
  // the window's edges: binades ebase and ebase + 13 are coded (1 and 14), ebase - 1 and ebase + 14 escape
  for (int ebase : {1, 900, 1010, 2033}) {
    for (int e = ebase - 1; e <= ebase + kCodes; ++e) {
      if (e < 1 || e > 2046) continue;
      for (uint64_t m : {0ull, 1ull, 0x000FFFFFFFFFFFFFull, 0x0000000080000000ull}) {
        for (uint64_t sgn : {0ull, 0x8000000000000000ull}) {
          const double v = double_of(sgn | ((uint64_t)e << 52) | m);
          const unsigned code = code_of(v, ebase);
          expect(e < ebase || e > ebase + kCodes - 1 ? code == kEscape : code == (unsigned)(e - ebase + 1), "edge code");
          for (unsigned c : cols) round_trip(v, c, ebase, esc);
        }
      }
    }
  }
  // zeros are code 0 and never escape; the all-zero word (slab padding) decodes to +0.0 at column 0
  expect(code_of(0.0, 1013) == 0u && code_of(-0.0, 1013) == 0u, "zero code");
  expect(bits_of(decode_value(0ull, nullptr, 1013)) == 0ull && decode_col(0u, 0u) == 0u, "padding word");
  // pick_ebase: the densest 14-binade window, clamped so that the window stays inside the normal exponents
  {
    std::vector<long long> h(2048, 0);
    for (int e = 990; e <= 1026; ++e) h[e] = 1;
    for (int e = 1000; e <= 1013; ++e) h[e] = 100;
    expect(pick_ebase(h.data()) == 1000, "pick_ebase interior");
    std::fill(h.begin(), h.end(), 0); h[2046] = 5;
    expect(pick_ebase(h.data()) == 2033, "pick_ebase top");
    std::fill(h.begin(), h.end(), 0); h[1] = 5;
    expect(pick_ebase(h.data()) == 1, "pick_ebase bottom");
    std::fill(h.begin(), h.end(), 0);
    for (int it = 0; it < 200; ++it) h[1 + next_u64() % 2046] += (long long)(next_u64() % 1000);
    long long best = -1; int arg = 0;
    for (int b = 1; b + kCodes - 1 <= 2046; ++b) {
      long long c = 0;
      for (int e = b; e < b + kCodes; ++e) c += h[e];
      if (c > best) { best = c; arg = b; }
    }
    expect(pick_ebase(h.data()) == arg, "pick_ebase brute force");
  }
  printf("checked %lld entries, bad %lld\n", n_checked, bad);
  return bad == 0 ? 0 : 1;
}
