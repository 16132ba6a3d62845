// sjb200_double.cuh -- element::get_double of one JSON Pointer result (sjb200_column_double_dev): the correctly rounded
// binary64 of a number's text, written once for the sm_90a kernels of sjb200_column_double.cu and for the host
// (tests/double_emul.cpp runs the same source under the host SIMT emulation).
//
// A number [s, e) of the input is read through a byte source (SpanSrc: byte i of the span, 0 past it) in three steps:
//   summarize  the shape of the text by a group of threads (SerialGroup: one lane; a warp or a CTA group of
//              sjb200_pointer.cuh for long numbers): where the '.', the 'e' and the first non-zero digit are, the exponent
//              (more than 18 significant exponent digits saturate at 999 999 999 999 999 999, as the reference's
//              parse_exponent does), and whether a non-zero digit follows the kMaxDigits-th significant digit.  Each
//              thread keeps the first position of each kind it sees and the group reduces with min, so a long number costs
//              one pass per group, not per lane.  Each thread reads runs of kRun consecutive bytes (rank * kRun, ...), so
//              that a thread has kRun independent loads in flight.
//   convert    the Clinger fast path (w <= 2^53, |q| <= 22: one correctly rounded __dmul_rn / __ddiv_rn), else the
//              Eisel-Lemire step: the first 19 significant digits w times the 128-bit power of five T_q of
//              sjb200_pow5.h.  T_q is 5^q truncated, so the exact product lies within 2 units of the product's top 128
//              bits; a result whose bits below the rounding point are within 3 units of the halfway point is
//              inconclusive.  With more than 19 digits, w and w + 1 must round alike.
//   exact      the inconclusive rows: the candidate b (the Eisel-Lemire product rounded down) or b + 1 ulp, decided by
//              comparing the decimal D * 10^e with the halfway point (2m + 1) * 2^(h) as big integers.  Only the first
//              kMaxDigits significant digits enter D; the others are a sticky bit (a halfway point of binary64 has at
//              most 767 significant digits, so they can only break a tie).
#pragma once
#include <stdint.h>

#include "sjb200_column.cuh"
#include "sjb200_pow5.h"

namespace sjb200 {
namespace dbl {

constexpr int32_t kNumberError = 9;         // simdjson::NUMBER_ERROR
constexpr int32_t kSlow = -1;               // convert: inconclusive, decide with exact()
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr uint32_t kMaxDigits = 768;        // significant digits that enter the exact comparison
constexpr int kLimbs = 90;                  // 32-bit limbs of a big integer of exact(): 2 880 bits
constexpr uint32_t kRun = 16;               // consecutive bytes a thread of summarize() reads per step
constexpr uint64_t kInfBits = 0x7FF0000000000000ull;
constexpr uint64_t kSignBit = 0x8000000000000000ull;

#if defined(__CUDACC__)
__device__ const uint64_t kPow5[] = {SJB200_POW5_WORDS};
__device__ const int16_t kPow5Shift[] = {SJB200_POW5_SHIFTS};
__device__ const double kPow10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11,
                                      1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
#else
static const uint64_t kPow5[] = {SJB200_POW5_WORDS};
static const int16_t kPow5Shift[] = {SJB200_POW5_SHIFTS};
static const double kPow10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11,
                                  1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
#endif

#if defined(__CUDA_ARCH__)
SJ_DEV uint64_t pow5_word(int i) { return __ldg(kPow5 + i); }
SJ_DEV int pow5_shift(int i) { return __ldg(kPow5Shift + i); }
SJ_DEV double pow10(int i) { return __ldg(kPow10 + i); }
SJ_DEV uint64_t mulhi(uint64_t a, uint64_t b) { return __umul64hi(a, b); }
SJ_DEV int clz64(uint64_t x) { return __clzll((long long)x); }
SJ_DEV double dmul(double a, double b) { return __dmul_rn(a, b); }
SJ_DEV double ddiv(double a, double b) { return __ddiv_rn(a, b); }
SJ_DEV double u64_to_double(uint64_t v) { return __ull2double_rn(v); }
SJ_DEV double i64_to_double(int64_t v) { return __ll2double_rn(v); }
SJ_DEV uint64_t bits_of(double d) { return uint64_t(__double_as_longlong(d)); }
#else
SJ_DEV uint64_t pow5_word(int i) { return kPow5[i]; }
SJ_DEV int pow5_shift(int i) { return kPow5Shift[i]; }
SJ_DEV double pow10(int i) { return kPow10[i]; }
SJ_DEV uint64_t mulhi(uint64_t a, uint64_t b) { return uint64_t((unsigned __int128)a * b >> 64); }
SJ_DEV int clz64(uint64_t x) { return __builtin_clzll(x); }
SJ_DEV double dmul(double a, double b) { return a * b; }  // (one operation: nothing to contract)
SJ_DEV double ddiv(double a, double b) { return a / b; }
SJ_DEV double u64_to_double(uint64_t v) { return double(v); }
SJ_DEV double i64_to_double(int64_t v) { return double(v); }
SJ_DEV uint64_t bits_of(double d) { uint64_t b; __builtin_memcpy(&b, &d, 8); return b; }
#endif

// Byte i of a span of the input, 0 past its end: nothing outside [p, p + len) is read.
struct SpanSrc {
  const uint8_t *p;
  uint32_t len;
  SJ_DEV uint32_t operator()(uint32_t i) const { return i < len ? sj_ldg_u8(p + i) : 0u; }
};

// One thread as the group of summarize().
struct SerialGroup {
  static constexpr unsigned kWidth = 1;
  SJ_DEV unsigned rank() const { return 0; }
  SJ_DEV int scan(int x, int *total) const { *total = x; return 0; }
  SJ_DEV uint32_t min(uint32_t x) const { return x; }
};

// The shape of a number's text (positions relative to the span's start).
struct Num {
  bool valid;     // the span is a JSON number: -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?
  bool neg;
  bool sticky;    // a non-zero digit after the kMaxDigits-th significant digit
  uint32_t nz;    // the first non-zero digit of the mantissa, kNone when the mantissa is zero
  uint32_t dot;   // the '.', kNone without one
  uint32_t mend;  // one past the mantissa: the 'e' / 'E', or the span's length
  int64_t exp;    // the exponent's value
};

SJ_DEV bool is_nonzero_digit(uint32_t c) { return c - '1' < 9u; }
SJ_DEV uint32_t cap2(uint32_t x) { return x < 2u ? x : 2u; }

// The summary of the span [0, L) by group g.  Every thread of the group calls it and gets the same result.
template <class G, class S>
SJ_DEV Num summarize(G &g, const S &at, uint32_t L) {
  uint32_t dot = kNone, ex = kNone, sign = kNone, nz = kNone, bad = kNone, ndot = 0, nex = 0, nsign = 0;
  for (uint64_t b = uint64_t(g.rank()) * kRun; b < L; b += uint64_t(G::kWidth) * kRun) {
#pragma unroll
    for (uint32_t j = 0; j < kRun; j++) {
      const uint32_t i = uint32_t(b) + j;
      if (i >= L) break;
      const uint32_t c = at(i);
      if (c - '0' < 10u) {
        if (nz == kNone && c != '0') nz = i;
      } else if (c == '.') {
        if (dot == kNone) dot = i;
        ndot = cap2(ndot + 1);
      } else if ((c | 0x20u) == 'e') {
        if (ex == kNone) ex = i;
        nex = cap2(nex + 1);
      } else if ((c == '-' || c == '+') && !(i == 0 && c == '-')) {
        if (sign == kNone) sign = i;
        nsign = cap2(nsign + 1);
      } else if (c != '-' && bad == kNone) {
        bad = i;
      }
    }
  }
  int t;
  g.scan(int(ndot), &t);
  const uint32_t dots = uint32_t(t);
  g.scan(int(nex), &t);
  const uint32_t exs = uint32_t(t);
  g.scan(int(nsign), &t);
  const uint32_t signs = uint32_t(t);
  dot = g.min(dot);
  ex = g.min(ex);
  sign = g.min(sign);
  nz = g.min(nz);
  bad = g.min(bad);
  Num m;
  m.neg = L > 0 && at(0) == '-';
  m.dot = dot;
  m.mend = ex == kNone ? L : ex;
  m.nz = nz < m.mend ? nz : kNone;
  m.sticky = false;
  m.exp = 0;
  const uint32_t ms = m.neg ? 1u : 0u;
  const uint32_t int_end = dot != kNone ? dot : m.mend;
  uint32_t es = ex == kNone ? L : ex + 1;
  if (ex != kNone && signs == 1 && sign == ex + 1) es++;
  m.valid = L > 0 && bad == kNone && dots <= 1 && exs <= 1 && (dot == kNone || dot + 1 < m.mend) && ms < int_end &&
            !(at(ms) == '0' && int_end - ms > 1) && (signs == 0 || (signs == 1 && ex != kNone && sign == ex + 1)) &&
            (ex == kNone || es < L);
  if (!m.valid || m.nz == kNone) return m;  // (uniform: every thread holds the same reductions)
  // the tail past the kMaxDigits-th significant digit (the sticky bit) and the exponent's first non-zero digit
  const uint32_t nd = m.mend - m.nz - (dot != kNone && dot > m.nz ? 1u : 0u);
  uint32_t tail = m.mend;
  if (nd > kMaxDigits) tail = m.nz + kMaxDigits + (dot != kNone && dot > m.nz && dot <= m.nz + kMaxDigits ? 1u : 0u);
  const uint32_t lo = tail < es ? tail : es;
  uint32_t sticky = 1, ez = kNone;
  for (uint64_t b = lo + uint64_t(g.rank()) * kRun; b < L; b += uint64_t(G::kWidth) * kRun) {
#pragma unroll
    for (uint32_t j = 0; j < kRun; j++) {
      const uint32_t i = uint32_t(b) + j;
      if (i >= L || !is_nonzero_digit(at(i))) continue;
      if (i < m.mend) {
        sticky = 0;
      } else if (i >= es && ez == kNone) {
        ez = i;
      }
    }
  }
  m.sticky = g.min(sticky) == 0;
  ez = g.min(ez);
  if (ez != kNone) {
    int64_t e = 999999999999999999ll;  // more than 18 significant digits (numberparsing.h parse_exponent)
    if (L - ez <= 18) {
      e = 0;
      for (uint32_t i = ez; i < L; i++) e = e * 10 + int64_t(at(i) - '0');
    }
    m.exp = at(ex + 1) == '-' ? -e : e;
  }
  return m;
}

// significant digits and the decimal exponent of D, the integer of all of them: the value is D * 10^dec_exp
SJ_DEV uint32_t sig_digits(const Num &m) { return m.mend - m.nz - (m.dot != kNone && m.dot > m.nz ? 1u : 0u); }
SJ_DEV int64_t dec_exp(const Num &m) { return m.exp - int64_t(m.dot != kNone ? m.mend - m.dot - 1 : 0u); }

// the first k significant digits as an integer (k <= 19)
template <class S>
SJ_DEV uint64_t leading_digits(const Num &m, const S &at, uint32_t k) {
  uint64_t w = 0;
  uint32_t p = m.nz;
  for (uint32_t j = 0; j < k; j++, p++) {
    if (p == m.dot) p++;
    w = w * 10u + (at(p) - '0');
  }
  return w;
}

// Eisel-Lemire on w * 10^q, q in [SJB200_POW5_QMIN, SJB200_POW5_QMAX]: *floor_bits = the bits of the value rounded down
// at its precision (the candidate of exact()).  Returns 1 to round up, 0 to keep the floor, -1 inconclusive;
// *floor_bits = kInfBits (return 0) when the value is at least 2^1024.
SJ_DEV int lemire(uint64_t w, int q, uint64_t *floor_bits) {
  const int idx = q - SJB200_POW5_QMIN;
  const uint64_t th = pow5_word(2 * idx), tl = pow5_word(2 * idx + 1);
  const int lz = clz64(w);
  const uint64_t wn = w << lz;
  // P = wn * T, 192 bits; its top 128 bits p2:p1 (the low word only moves them by a carry, taken as uncertainty)
  const uint64_t a_hi = mulhi(wn, tl);
  const uint64_t b_lo = wn * th, b_hi = mulhi(wn, th);
  const uint64_t p1 = b_lo + a_hi;
  const uint64_t p2 = b_hi + (p1 < b_lo ? 1u : 0u);
  const int upper = int(p2 >> 63);
  const int E = 190 + upper + q + pow5_shift(idx) - lz + 1023;  // the biased exponent of the leading bit
  if (E >= 2047) {
    *floor_bits = kInfBits;
    return 0;
  }
  const int s = 74 + upper + (E < 1 ? 1 - E : 0);  // bits of p2:p1 below the result's last bit
  if (s >= 128) {  // below 2^-1074: 0 or the least subnormal
    *floor_bits = 0;
    return -1;
  }
  const int sh = s - 64;  // in [10, 63]
  const uint64_t m = p2 >> sh;
  const uint64_t rh = p2 & ((1ull << sh) - 1u), hh = 1ull << (sh - 1);  // the remainder's and the halfway point's high words
  *floor_bits = (uint64_t(E < 1 ? 0 : E - 1) << 52) + m;
  if (rh == hh) return p1 <= 3u ? -1 : 1;
  if (rh == hh - 1u) return p1 >= ~3ull ? -1 : 0;
  return rh > hh ? 1 : 0;
}

// ---- the exact comparison: little-endian 32-bit limbs, limb i of a number at x[i * stride]
struct Big {
  uint32_t *x;
  unsigned stride;
  int n;  // limbs in use
  SJ_DEV uint32_t &operator[](int i) { return x[unsigned(i) * stride]; }
};
SJ_DEV void big_set(Big &b, uint64_t v) {
  b[0] = uint32_t(v);
  b[1] = uint32_t(v >> 32);
  b.n = b[1] ? 2 : 1;
}
SJ_DEV void big_mul_add(Big &b, uint32_t f, uint32_t add) {
  uint64_t carry = add;
  for (int i = 0; i < b.n; i++) {
    const uint64_t v = uint64_t(b[i]) * f + carry;
    b[i] = uint32_t(v);
    carry = v >> 32;
  }
  if (carry && b.n < kLimbs) b[b.n++] = uint32_t(carry);
}
SJ_DEV void big_mul_pow5(Big &b, uint32_t e) {
  for (; e >= 13; e -= 13) big_mul_add(b, 1220703125u, 0);  // 5^13
  uint32_t f = 1;
  for (; e; e--) f *= 5u;
  if (f != 1) big_mul_add(b, f, 0);
}
SJ_DEV void big_shl(Big &b, uint32_t bits) {
  const int limbs = int(bits >> 5), r = int(bits & 31u);
  int n = b.n + limbs + 1;
  if (n > kLimbs) n = kLimbs;  // (the bounds of exact() keep every number below kLimbs limbs)
  for (int i = n - 1; i >= 0; i--) {
    const int j = i - limbs;
    const uint32_t hi = j >= 0 && j < b.n ? b[j] : 0u, lo = j - 1 >= 0 && j - 1 < b.n ? b[j - 1] : 0u;
    b[i] = r ? (hi << r) | (lo >> (32 - r)) : hi;
  }
  while (n > 1 && b[n - 1] == 0) n--;
  b.n = n;
}
SJ_DEV int big_cmp(Big &a, Big &b) {
  if (a.n != b.n) return a.n > b.n ? 1 : -1;
  for (int i = a.n - 1; i >= 0; i--)
    if (a[i] != b[i]) return a[i] > b[i] ? 1 : -1;
  return 0;
}

// The inconclusive row: floor_bits (lemire() of the first 19 digits) or the next double, by D * 10^e against the halfway
// point between them.  a, b: kLimbs limbs each.  Returns the value's bits (kInfBits and up: infinite), sign not applied.
template <class S>
SJ_DEV uint64_t exact(const Num &m, const S &at, uint64_t floor_bits, Big a, Big b) {
  const uint32_t nd = sig_digits(m);
  const uint32_t nk = nd < kMaxDigits ? nd : kMaxDigits;
  const int64_t e10 = dec_exp(m) + int64_t(nd - nk);  // in [-1091, 308] (convert() ruled out the rest)
  // A = the first nk digits, nine at a time
  big_set(a, 0);
  uint32_t p = m.nz, chunk = 0, f = 1;
  for (uint32_t j = 0; j < nk; j++, p++) {
    if (p == m.dot) p++;
    chunk = chunk * 10u + (at(p) - '0');
    f *= 10u;
    if (f == 1000000000u || j + 1 == nk) {
      big_mul_add(a, f, chunk);
      chunk = 0;
      f = 1;
    }
  }
  // the halfway point (2 mb + 1) * 2^(h)
  const uint32_t ef = uint32_t(floor_bits >> 52);
  const uint64_t mb = (floor_bits & ((1ull << 52) - 1u)) | (ef ? 1ull << 52 : 0u);
  const int64_t h = (ef ? int64_t(ef) - 1075 : -1074) - 1;
  big_set(b, 2 * mb + 1);
  if (e10 >= 0)
    big_mul_pow5(a, uint32_t(e10));
  else
    big_mul_pow5(b, uint32_t(-e10));
  // compare A * 2^e10 with B * 2^h
  if (e10 > h)
    big_shl(a, uint32_t(e10 - h));
  else if (h > e10)
    big_shl(b, uint32_t(h - e10));
  int c = big_cmp(a, b);
  if (c == 0 && m.sticky) c = 1;
  return c > 0 || (c == 0 && (floor_bits & 1u)) ? floor_bits + 1 : floor_bits;
}

// The value of a summarized number: 0 with *bits, kNumberError (infinite), or kSlow with *floor_bits for exact().
template <class S>
SJ_DEV int32_t convert(const Num &m, const S &at, uint64_t *bits, uint64_t *floor_bits) {
  const uint64_t sign = m.neg ? kSignBit : 0u;
  *bits = sign;
  if (m.nz == kNone) return 0;  // (-)0.0
  const uint32_t nd = sig_digits(m);
  const uint32_t k = nd < 19u ? nd : 19u;
  const int64_t q = dec_exp(m) + int64_t(nd - k);
  if (q < SJB200_POW5_QMIN) return 0;  // below 10^19 * 10^-343: rounds to zero
  if (q > SJB200_POW5_QMAX) return kNumberError;  // at least 10^309
  const uint64_t w = leading_digits(m, at, k);
  if (nd <= 19 && w <= (1ull << 53) && q >= -22 && q <= 22) {  // Clinger: both operands exact, one rounding
    const double d = u64_to_double(w);
    *bits = sign | bits_of(q >= 0 ? dmul(d, pow10(int(q))) : ddiv(d, pow10(int(-q))));
    return 0;
  }
  uint64_t fb;
  int dir = lemire(w, int(q), &fb);
  *floor_bits = fb;
  if (dir >= 0 && nd > 19) {  // the digits past the 19th: w + 1 must round alike
    uint64_t fb1;
    const int dir1 = lemire(w + 1, int(q), &fb1);
    if (dir1 < 0 || fb1 + uint64_t(dir1) != fb + uint64_t(dir)) dir = -1;
  }
  if (dir < 0) return kSlow;
  const uint64_t v = fb + uint64_t(dir);
  if (v >= kInfBits) return kNumberError;
  *bits = sign | v;
  return 0;
}

// The row's value after exact(): 0 with *bits, or kNumberError
SJ_DEV int32_t finish_exact(const Num &m, uint64_t v, uint64_t *bits) {
  *bits = 0;
  if (v >= kInfBits) return kNumberError;
  *bits = (m.neg ? kSignBit : 0u) | v;
  return 0;
}

// get_double of an integer token (element-inl.h: double(int64) / double(uint64), round to nearest even)
SJ_DEV uint64_t integer_bits(uint32_t t, uint64_t v) { return bits_of(t == 'u' ? u64_to_double(v) : i64_to_double(int64_t(v))); }

}  // namespace dbl
}  // namespace sjb200
