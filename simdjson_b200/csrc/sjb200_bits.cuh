// sjb200_bits.cuh -- the per-lane bit-plane arithmetic of the H100 stage-1 kernels.
//
// Everything in this header is a pure function of its arguments (no warp
// intrinsics, no memory), compiled for both host and device, so that the
// algebra can be unit-tested on a CPU (tests/host_emul.cpp) while the CUDA
// kernels (sjb200_kernels.cu) add only the data movement and the
// warp / CTA / grid carry plumbing around it.
//
// Formulation (NOT the reference's: it classifies bytes with 64-byte SIMD
// shuffles, src/icelake.cpp L48-96): a lane transposes 32 input bytes into
// eight 32-bit *bit planes* (plane k, bit n = bit k of byte n).  Every
// character class, the UTF-8 rules and the string/scalar logic are then plain
// boolean functions of planes, 32 bytes per LOP3.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SJ_HD __host__ __device__ __forceinline__
#else
#define SJ_HD inline
#endif

namespace sjb200 {

// ---------------------------------------------------------------- helpers
SJ_HD uint32_t byte_perm(uint32_t x, uint32_t y, uint32_t s) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(x, y, s);
#else
  uint64_t pool = (uint64_t(y) << 32) | x;
  uint32_t r = 0;
  for (int i = 0; i < 4; i++) {
    uint32_t sel = (s >> (4 * i)) & 7;
    r |= uint32_t((pool >> (8 * sel)) & 0xFF) << (8 * i);
  }
  return r;
#endif
}
SJ_HD int popc32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}
SJ_HD int ctz32(uint32_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
  return __ffs(x) - 1;
#else
  return __builtin_ctz(x);
#endif
}
// (cur << n) | (prev >> (32-n)), 1 <= n <= 3: shift a mask towards higher byte
// positions, pulling the top bits of the previous 32-byte unit in.
SJ_HD uint32_t shl_in(uint32_t prev, uint32_t cur, int n) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_l(prev, cur, n);
#else
  return (cur << n) | (prev >> (32 - n));
#endif
}

// (a & m) | (b & ~m) -- one LOP3 (the compiler otherwise splits the two constant masks into two)
SJ_HD uint32_t bitsel(uint32_t m, uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(d) : "r"(a), "r"(b), "r"(m));
  return d;
#else
  return (a & m) | (b & ~m);
#endif
}

// x >> d for a constant d, on the FMA pipe (IMAD.HI) instead of the ALU pipe (SHF): the scan is bound by the ALU pipe's
// issue rate, the FMA pipe is mostly idle.  Build option; the multiply is slower per instruction, so it only pays if
// it overlaps (compare the two builds).
#ifndef SJB200_SHR_IMAD
#define SJB200_SHR_IMAD 0
#endif
template <int D>
SJ_HD uint32_t shr_const(uint32_t x) {
#if defined(__CUDA_ARCH__) && SJB200_SHR_IMAD
  uint32_t r;
  asm("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(x), "n"(1u << (32 - D)));
  return r;
#else
  return x >> D;
#endif
}

// ------------------------------------------------------------- transpose
// w[i] (i=0..7) holds input bytes 4i..4i+3 little-endian.  On return p[k] bit n
// = bit k of byte n (n = 0..31).
//   step 1: two 4x4 byte transposes (16 PRMT): a[r] byte j = input byte 8j+r
//   step 2: 8x8 bit-matrix transpose inside every byte lane (3 delta-swap
//           stages x 4 register pairs x {2 shifts + 2 LOP3})
SJ_HD void transpose32(const uint32_t w[8], uint32_t p[8]) {
  uint32_t t0 = byte_perm(w[0], w[2], 0x5140), t1 = byte_perm(w[0], w[2], 0x7362);
  uint32_t t2 = byte_perm(w[4], w[6], 0x5140), t3 = byte_perm(w[4], w[6], 0x7362);
  uint32_t a0 = byte_perm(t0, t2, 0x5410), a1 = byte_perm(t0, t2, 0x7632);
  uint32_t a2 = byte_perm(t1, t3, 0x5410), a3 = byte_perm(t1, t3, 0x7632);
  t0 = byte_perm(w[1], w[3], 0x5140); t1 = byte_perm(w[1], w[3], 0x7362);
  t2 = byte_perm(w[5], w[7], 0x5140); t3 = byte_perm(w[5], w[7], 0x7362);
  uint32_t a4 = byte_perm(t0, t2, 0x5410), a5 = byte_perm(t0, t2, 0x7632);
  uint32_t a6 = byte_perm(t1, t3, 0x5410), a7 = byte_perm(t1, t3, 0x7632);
#define SJ_DSWAP(lo, hi, d, m)                      \
  {                                                 \
    const uint32_t nl = bitsel(m, lo, (hi) << (d)); \
    const uint32_t nh = bitsel(m, shr_const<d>(lo), hi); \
    lo = nl; hi = nh;                               \
  }
  SJ_DSWAP(a0, a1, 1, 0x55555555u) SJ_DSWAP(a2, a3, 1, 0x55555555u)
  SJ_DSWAP(a4, a5, 1, 0x55555555u) SJ_DSWAP(a6, a7, 1, 0x55555555u)
  SJ_DSWAP(a0, a2, 2, 0x33333333u) SJ_DSWAP(a1, a3, 2, 0x33333333u)
  SJ_DSWAP(a4, a6, 2, 0x33333333u) SJ_DSWAP(a5, a7, 2, 0x33333333u)
  SJ_DSWAP(a0, a4, 4, 0x0F0F0F0Fu) SJ_DSWAP(a1, a5, 4, 0x0F0F0F0Fu)
  SJ_DSWAP(a2, a6, 4, 0x0F0F0F0Fu) SJ_DSWAP(a3, a7, 4, 0x0F0F0F0Fu)
#undef SJ_DSWAP
  p[0] = a0; p[1] = a1; p[2] = a2; p[3] = a3; p[4] = a4; p[5] = a5; p[6] = a6; p[7] = a7;
}

// --------------------------------------------------------- character classes
// One 32-byte unit's class masks.  Character sets are the reference's x86 ones
// (src/icelake.cpp L48-96, src/generic/json_character_block.h L12-22):
//   whitespace {20,09,0A,0D};  op {2C,3A,5B,5D,7B,7D} + {0C,1A} (the |0x20 quirk);
//   scalar = ~(op|ws);  ctl = byte <= 0x1F (json_structural_indexer.h L240).
struct unit_classes {
  uint32_t bs;   // '\\'
  uint32_t qu;   // '"' (raw, before escape masking)
  uint32_t op;
  uint32_t sc;   // scalar
  uint32_t ctl;  // < 0x20
};

SJ_HD unit_classes classify(const uint32_t p[8]) {
  const uint32_t b0 = p[0], b1 = p[1], b2 = p[2], b3 = p[3], b4 = p[4], b5 = p[5], b6 = p[6], b7 = p[7];
  unit_classes c;
  c.ctl = ~b7 & ~b6 & ~b5;                      // 000x xxxx
  const uint32_t u = ~b7 & ~b6 & b5;            // 001x xxxx
  const uint32_t v = ~b4 & ~b3 & ~b2;           // xxx0 00xx
  const uint32_t z = ~b1 & ~b0;                 // xxxx xx00
  c.qu = u & v & (b1 & ~b0);                    // 0010 0010
  c.bs = (~b7 & b6 & ~b5) & (b4 & b3 & b2) & z; // 0101 1100
  const uint32_t sp = u & v & z;                // 0010 0000
  // 09, 0A, 0D : 0000 1xxx with low3 in {001,010,101}
  const uint32_t low3 = (~b2 & (b1 ^ b0)) | (b2 & ~b1 & b0);
  const uint32_t ws = sp | (c.ctl & ~b4 & b3 & low3);
  // operators, bit 5 is don't-care: x0x0 1100 (0C 2C), x0x1 1010 (1A 3A), x1x1 1011 (5B 7B), x1x1 1101 (5D 7D)
  const uint32_t pA = b2 & ~b1 & ~b0, pB = ~b2 & b1 & ~b0, pCD = (~b2 & b1 & b0) | (b2 & ~b1 & b0);
  const uint32_t sel = (~b6 & ~b4 & pA) | (~b6 & b4 & pB) | (b6 & b4 & pCD);
  c.op = ~b7 & b3 & sel;
  c.sc = ~(c.op | ws);
  return c;
}

// -------------------------------------------------------------------- utf-8
// Lead-byte masks of one unit that the next unit needs (their top 3 bits).
struct utf8_carry {
  uint32_t n1;  // bytes that need a continuation 1 later  (>= C0)
  uint32_t n2;  // ... 2 later (>= E0)
  uint32_t n3;  // ... 3 later (>= F0)
  uint32_t e0, ed, f0, f4;  // leads with a constrained second byte
};
SJ_HD utf8_carry utf8_carry_zero() {
  utf8_carry c;
  c.n1 = c.n2 = c.n3 = c.e0 = c.ed = c.f0 = c.f4 = 0;
  return c;
}
SJ_HD bool utf8_carry_pending(const utf8_carry &c) { return ((c.n1 >> 31) | (c.n2 >> 30) | (c.n3 >> 29)) != 0; }

// Carry for the first unit of a lane from the 4 bytes that precede it
// (little-endian word: byte -1 is the top byte).  Bytes that are themselves
// invalid (C0,C1,F5..FF) are flagged where they are classified, so ">= F0"
// style tests are sufficient here.
SJ_HD utf8_carry utf8_carry_from_prev_word(uint32_t pw) {
  utf8_carry c = utf8_carry_zero();
  if ((pw & 0x80808000u) == 0) return c;
  const uint32_t m1 = pw >> 24, m2 = (pw >> 16) & 0xFF, m3 = (pw >> 8) & 0xFF;
  c.n1 = uint32_t(m1 >= 0xC0) << 31;
  c.n2 = (uint32_t(m1 >= 0xE0) << 31) | (uint32_t(m2 >= 0xE0) << 30);
  c.n3 = (uint32_t(m1 >= 0xF0) << 31) | (uint32_t(m2 >= 0xF0) << 30) | (uint32_t(m3 >= 0xF0) << 29);
  c.e0 = uint32_t(m1 == 0xE0) << 31;
  c.ed = uint32_t(m1 == 0xED) << 31;
  c.f0 = uint32_t(m1 == 0xF0) << 31;
  c.f4 = uint32_t(m1 == 0xF4) << 31;
  return c;
}

// Validate one 32-byte unit given the previous unit's carry; returns a mask
// that is non-zero iff some byte of this unit violates UTF-8 well-formedness
// (Unicode table 3-7: the same boolean utf8_lookup4_algorithm.h L145-202
// computes; see SURVEY.md 8(a) equivalence note).  `carry` is updated.
// A sequence truncated by the end of the unit is reported by the *next* unit
// (or by the end-of-input check), through the carry.
SJ_HD uint32_t utf8_check_unit(const uint32_t p[8], utf8_carry &carry) {
  const uint32_t b0 = p[0], b1 = p[1], b2 = p[2], b3 = p[3], b4 = p[4], b5 = p[5], b6 = p[6], b7 = p[7];
  const uint32_t cont = b7 & ~b6;
  const uint32_t l234 = b7 & b6;          // >= C0
  const uint32_t l34 = l234 & b5;         // >= E0
  const uint32_t l4x = l34 & b4;          // >= F0
  const uint32_t l2 = l234 & ~b5;
  const uint32_t l3 = l34 & ~b4;
  uint32_t err = l4x & b3;                               // F8..FF
  err |= l2 & ~b4 & ~b3 & ~b2 & ~b1;                     // C0, C1
  err |= l4x & b2 & (b1 | b0);                           // F5..F7
  const uint32_t lo4z = ~b3 & ~b2 & ~b1 & ~b0;
  utf8_carry cur;
  cur.n1 = l234; cur.n2 = l34; cur.n3 = l4x;
  cur.e0 = l3 & lo4z;                                    // E0
  cur.ed = l3 & b3 & b2 & ~b1 & b0;                      // ED
  cur.f0 = l4x & lo4z;                                   // F0  (F8.. already flagged)
  cur.f4 = l4x & ~b3 & b2 & ~b1 & ~b0;                   // F4
  const uint32_t expect = shl_in(carry.n1, cur.n1, 1) | shl_in(carry.n2, cur.n2, 2) | shl_in(carry.n3, cur.n3, 3);
  err |= expect ^ cont;                                  // missing or stray continuation
  err |= shl_in(carry.e0, cur.e0, 1) & ~b5;              // E0 80..9F  overlong
  err |= shl_in(carry.ed, cur.ed, 1) & b5;               // ED A0..BF  surrogates
  err |= shl_in(carry.f0, cur.f0, 1) & ~b5 & ~b4;        // F0 80..8F  overlong
  err |= shl_in(carry.f4, cur.f4, 1) & (b5 | b4);        // F4 90..BF  > U+10FFFF
  carry = cur;
  return err;
}

// ---------------------------------------------------------------- escapes
// json_escape_scanner::next (json_escape_scanner.h L50-71, L96-143) widened
// from one 64-bit block to W 32-bit words and evaluated with carry-in 0.
// escaped[u] = bytes preceded by an odd-length backslash run.  Returns the
// carry-out (last byte is an unescaped backslash).
template <int W>
SJ_HD uint32_t escape_scan(const uint32_t bs[W], uint32_t escaped[W]) {
  const uint32_t ODD = 0xAAAAAAAAu;
  uint32_t borrow = 0, escape_last = 0;
#pragma unroll
  for (int u = 0; u < W; u++) {
    const uint32_t maybe = u ? shl_in(bs[u - 1], bs[u], 1) : (bs[u] << 1);
    const uint32_t x = maybe | ODD;
    const uint64_t d = uint64_t(x) - uint64_t(bs[u]) - uint64_t(borrow);
    borrow = uint32_t(d >> 32) & 1u;
    const uint32_t eatc = uint32_t(d) ^ ODD;
    escaped[u] = eatc ^ bs[u];
    escape_last = eatc & bs[u];
  }
  return escape_last >> 31;
}

// number of leading backslashes of a lane chunk (0..32W)
template <int W>
SJ_HD int leading_backslashes(const uint32_t bs[W]) {
  int k = 0;
#pragma unroll
  for (int u = 0; u < W; u++) {
    if (k == 32 * u) k += (bs[u] == 0xFFFFFFFFu) ? 32 : ctz32(~bs[u]);
  }
  return k;
}

// prefix XOR over one word: bit i of the result = XOR of bits 0..i
// (the reference does this with a carry-less multiply: icelake/bitmask.h L18-24)
SJ_HD uint32_t prefix_xor32(uint32_t x) {
  x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
  return x;
}

// ------------------------------------------------ carry transducer (SURVEY 8a)
// The effect of a chunk on the scanner state as a function of the incoming
// escape bit e:  T(e) = (esc_out, quote parity, last byte is a non-quote scalar).
// Packed: bit0 esc(0), bit1 par(0), bit2 scal(0), bit3 esc(1), bit4 par(1), bit5 scal(1).
SJ_HD uint32_t tt_make(uint32_t esc0, uint32_t par0, uint32_t scal0, uint32_t esc1, uint32_t par1, uint32_t scal1) {
  return (esc0 & 1) | ((par0 & 1) << 1) | ((scal0 & 1) << 2) | ((esc1 & 1) << 3) | ((par1 & 1) << 4) | ((scal1 & 1) << 5);
}
// apply T to an incoming state (bit0 esc, bit1 in_string, bit2 prev_scalar) -> outgoing state
SJ_HD uint32_t tt_apply(uint32_t T, uint32_t state) {
  const uint32_t o = (state & 1) ? (T >> 3) & 7 : T & 7;
  return (o & 1) | ((((state >> 1) ^ (o >> 1)) & 1) << 1) | (o & 4);
}
// (newer o older): first `older`, then `newer`
SJ_HD uint32_t tt_compose(uint32_t newer, uint32_t older) {
  uint32_t r = 0;
#pragma unroll
  for (int e = 0; e < 2; e++) {
    const uint32_t a = e ? (older >> 3) & 7 : older & 7;
    const uint32_t b = (a & 1) ? (newer >> 3) & 7 : newer & 7;
    const uint32_t o = (b & 1) | (((a ^ b) & 2)) | (b & 4);
    r |= o << (3 * e);
  }
  return r;
}
// a chunk whose outgoing state is the constant `state` (used to seed look-back with an inclusive prefix)
SJ_HD uint32_t tt_const(uint32_t state) { return (state & 7) | ((state & 7) << 3); }

// ------------------------------------------------ boundary state from the bytes before a tile
// Two of the three scanner-state bits entering a tile can be read off the bytes just before it:
//   e = the tile's first byte is escaped      <=> an odd-length backslash run ends at byte -1
//   c = byte -1 is a "non-quote scalar"       (json_scanner.h L148-149: scalar and not an unescaped quote)
// p16[0..3] are the 16 bytes before the tile, little-endian words (byte -1 is the top byte of p16[3]).
// Returns bit0 e, bit2 c (same positions as the scanner state) and bit3 = UNKNOWN when the backslash
// run reaches the start of the 16 bytes (then only the look-back chain knows; the caller handles it).
// Only the third bit, in_string, genuinely needs the whole prefix.
SJ_HD uint32_t boundary_state_from_prev16(const uint32_t p16[4]) {
  auto byte_at = [&](int back) -> uint32_t {  // back = 1..16 : byte -back
    const int i = 16 - back;
    return (p16[i >> 2] >> (8 * (i & 3))) & 0xFFu;
  };
  const uint32_t last = byte_at(1);
  int run_from = (last == '"') ? 2 : 1;  // a quote's own status depends on the run before it
  int run = 0;
  while (run_from + run <= 16 && byte_at(run_from + run) == '\\') run++;
  const bool unknown = (run_from + run > 16);
  const uint32_t odd = run & 1;
  uint32_t e, c;
  if (last == '"') {
    e = 0;        // a quote never escapes what follows
    c = odd;      // escaped quote = scalar byte; real quote = not
  } else {
    e = odd;      // run ending at byte -1 (run == 0 when byte -1 is not a backslash)
    const bool ws = last == 0x20 || last == 0x09 || last == 0x0A || last == 0x0D;
    const bool op = last == 0x2C || last == 0x3A || last == 0x5B || last == 0x5D || last == 0x7B || last == 0x7D || last == 0x0C || last == 0x1A;
    c = (ws || op) ? 0u : 1u;
  }
  return e | (c << 2) | (unknown ? 8u : 0u);
}

// Resolve the escape carries of 32 consecutive lane chunks at once.
//   G bit i: lane i ends with an unescaped backslash (evaluated with carry-in 0)
//   P bit i: lane i is all backslashes (its carry-out equals its carry-in)
// returns carry-in of every lane for warp carry-in cin; *cout = warp carry-out.
// c[i+1] = G[i] | (P[i] & c[i]) is the carry chain of the addition (G|P) + G + cin.
SJ_HD uint32_t escape_carries(uint32_t G, uint32_t P, uint32_t cin, uint32_t *cout) {
  const uint64_t s = uint64_t(G | P) + uint64_t(G) + uint64_t(cin);
  *cout = uint32_t(s >> 32) & 1u;
  return uint32_t(s) ^ P;
}

}  // namespace sjb200
