// sjb200_scan4.cuh -- the stage-1 structural indexer, fourth generation ("scan4").
//
// What it replaces in the reference (CPU, 64-byte SIMD blocks, strictly serial carries):
//   json_structural_indexer::index<128> / step / next   src/generic/stage1/json_structural_indexer.h L193-247
//   json_scanner::next, json_string_scanner::next, json_escape_scanner::next
//                                                        json_scanner.h L134-157, json_string_scanner.h L62-85,
//                                                        json_escape_scanner.h L50-71
//   bit_indexer::write                                   json_structural_indexer.h L93-122 (src/icelake.cpp L129-160)
//   utf8_checker                                         utf8_lookup4_algorithm.h L145-202
//
// Design (GPU-first; nothing here resembles the reference's block loop):
//   * The document is cut into 4 KiB *blocks* (one TMA box of 32 rows x 128 B, 128B-swizzled, so lane L owns row L and
//     reads it with conflict-free LDS.128) and *elements* of kScanWarps consecutive blocks (64 KiB), one block per scan warp.
//   * A CTA is kScanWarps (16) independent *scan warps* + 1 *chain warp*, persistent, one CTA per SM, pulling elements
//     from an atomic ticket.  Scan warps never synchronise with each other: every block is scanned on its own.  Two of
//     the three scanner state bits entering a block (next-byte-is-escaped, previous-byte-is-a-scalar) are read off the
//     bytes before it; the third (in-string) needs the whole prefix, so a block is finished for BOTH polarities: two
//     candidate structural masks, two counts, one quote parity.  The masks wait ("are parked") until the block's
//     polarity and output offset are known.
//   * The last scan warp to finish an element composes its block summaries and publishes the element's aggregate
//     {parity, count0, count1} in a decoupled look-back chain (one 64-bit descriptor per element).
//   * The chain warp walks back 320 descriptors per round trip (k-major: 256 contiguous bytes per load instruction) to
//     the nearest inclusive prefix, folds them with ballots / popcounts / REDUX, publishes the element's inclusive
//     prefix and posts every block's polarity and output offset to the scan warps through an mbarrier.
//   * Software pipeline: a scan warp emits element j-2 after scanning element j (per-lane bit loops into a
//     shared-memory staging area -- the block buffer it has just consumed -- and coalesced 16-byte stores).  The TMA
//     load of its next block is always in flight.  A second schedule ("deferred": masks parked in an L2-resident
//     scratch ring, all emits after the CTA's last scan) is kept as an option.
//   * All arithmetic is the bit-plane algebra of sjb200_bits.cuh: 32 bytes per LOP3, no per-byte code.
//
// The same source compiles for the host SIMT emulation (SJB200_HOST_EMU, tests/simt_emul.cpp), which runs it with one
// OS thread per CUDA thread against the oracle on machines without a GPU.
#pragma once
#include "sjb200_bits.cuh"
#include "sjb200_params.h"
#include "sjb200_simt.cuh"

namespace sjb200 {
namespace scan4 {

#ifndef SJB200_SCAN4_WARPS
#define SJB200_SCAN4_WARPS 16
#endif
constexpr int kScanWarps = SJB200_SCAN4_WARPS;  // scan warps per CTA = blocks per element.  16 (one CTA per SM, 64 KiB elements) rather than
                                                // 8 (two CTAs per SM): half the chain warps polling the descriptors, half the elements to resolve
constexpr int kBlockBytes = 4096;
constexpr int kBlockRows = kBlockBytes / 128;
constexpr int kChainWarps = 1;  // the warp that resolves this CTA's elements
#ifndef SJB200_SCAN4_EMITW
#define SJB200_SCAN4_EMITW 0
#endif
// Emit warps (stage 1 only): the scan is bound by the ALU pipe, the emit by FLO / shared-memory latency.  When the warp
// that scanned a block also emits it, all warps of the CTA sit in the emit loop together, with the ALU pipe
// nearly idle.  Dedicated warps take resolved blocks from a CTA-wide queue
// and emit them while the scan warps go on scanning.  0: every scan warp emits its own blocks (minify always does).
constexpr int kEmitWarps = SJB200_SCAN4_EMITW;
constexpr int kThreads4 = 32 * (kScanWarps + kChainWarps + kEmitWarps);
#ifndef SJB200_SCAN4_PARK
#define SJB200_SCAN4_PARK 3
#endif
constexpr int kPark = SJB200_SCAN4_PARK;  // elements whose masks wait in shared memory: a scan warp emits element j-kLag after scanning j
constexpr int kLag = kPark - 1;
constexpr int kNS = 32;          // ring of element slots (tickets, summaries, resolutions)
constexpr int kParkSlotWords = 2 * kScanWarps * 32 * 4 + kScanWarps * 32;  // one element's parked words (both polarities + prefixes)
#ifndef SJB200_SCAN4_GPARK
#define SJB200_SCAN4_GPARK 8
#endif
// With emit warps the parked masks may wait in an L2-resident scratch ring in global memory (ScanParams::park) instead of
// shared memory: the emit warps do not care about the extra latency, and the ring can be deep -- the scan warps then
// never wait for the chain as long as an element is resolved and emitted within kGPark - 1 scans (with three elements
// parked in shared memory, every hiccup of the look-back chain stalled the scan).  0: park in shared memory.
constexpr int kGPark = (SJB200_SCAN4_EMITW > 0) ? SJB200_SCAN4_GPARK : 0;
constexpr int kParkRing = (kGPark > 0) ? kGPark : 1;  // slots per CTA of the global scratch ring
constexpr int kParkFree = (kGPark > 0) ? kGPark : kPark;   // elements whose masks may be parked at once (emit-warp mode)
#ifndef SJB200_SCAN4_LOOKK
#define SJB200_SCAN4_LOOKK 10
#endif
constexpr int kLookK = SJB200_SCAN4_LOOKK;       // descriptors per lane and look-back round trip (window of 320 elements >= one wave of CTAs)
static_assert(kLag >= 1 && 2 * kLag + 3 <= kNS && 2 * kGPark + 4 <= kNS && (kNS & (kNS - 1)) == 0, "slot ring");
#ifndef SJB200_SCAN4_TRACE
#define SJB200_SCAN4_TRACE 0  // 1: tuning build that records where a scan warp's time goes (shared memory, dumped to ScanParams::debug at exit)
#endif
constexpr int kTraceIters = 8, kTracePoints = 12;
#if SJB200_SCAN4_TRACE
#define SJ_TRACE4(pt)                                                                                              \
  do {                                                                                                             \
    if (lane == 0 && (warp == 0 || warp == 9) && j < uint32_t(kTraceIters)) S->trace[warp ? 1 : 0][j][pt] = sj_clock32(); \
  } while (0)
#else
#define SJ_TRACE4(pt) do { } while (0)
#endif
constexpr uint32_t kSpinLimit4 = 1u << 21;  // bounded waits: a stuck protocol becomes kFlagInternal, never a hang
constexpr uint32_t kStageWords = kBlockBytes / 4;
constexpr int kElemBytes = kScanWarps * kBlockBytes;  // 32 KiB or 64 KiB: what one CTA scans per ticket, one look-back descriptor
static_assert(kElemBytes % kTileBytes == 0 && kScanWarps <= 16, "an element is a whole number of tiles of the launch parameter block");
SJ_DEV uint32_t elements_of(const ScanParams &p) { return uint32_t((uint64_t(p.ntiles) * kTileBytes + kElemBytes - 1) / kElemBytes); }

enum : uint32_t { kDescNone = 0, kDescAgg = 1, kDescInc = 2 };

struct Smem {
  uint8_t ring[kScanWarps][2][kBlockBytes];   // per scan warp: two block buffers (TMA destination / emit staging)
  uint8_t estage[kEmitWarps > 0 ? kEmitWarps : 1][kBlockBytes];  // emit warps: staging areas (1 KiB aligned like the ring: minify fetches blocks into them by TMA)
  sj_u4 park[kGPark > 0 ? 1 : kPark][2][kGPark > 0 ? 1 : kScanWarps * 32];  // [pipeline buffer][polarity][thread]: candidate structural masks (shared-memory parking)
  uint32_t parkpre[kGPark > 0 ? 1 : kPark][kGPark > 0 ? 1 : kScanWarps * 32];  // exclusive prefix of the lane's counts inside its block, both polarities packed
  uint32_t compact_lut[16];                   // minify: see compact_entry
  uint32_t ticket[kNS];
  uint32_t summary[kNS][kScanWarps];          // c0 | c1<<16 | parity<<29 | ctl-hit0<<30 | ctl-hit1<<31
  uint32_t arrived[kNS];                      // scan warps done with the element (the last one composes and publishes)
  uint32_t elem[kNS][4];                      // composed element: quote parity, outputs entered outside / inside a string, ctl hits (bit0/1)
  uint32_t pre[kNS][2][kScanWarps];           // per block, for either polarity at the start of the element: polarity<<31 | outputs before it
  uint32_t res_pol[kNS][kScanWarps];          // in-string polarity entering the block
  uint32_t res_base[kNS][kScanWarps];         // outputs of this launch before the block
  sj_mbar_t full[kScanWarps][2];
  sj_mbar_t ticket_ready[kNS];
  sj_mbar_t scanned[kNS];
  sj_mbar_t resolved[kNS];
  // emit warps
  sj_mbar_t efull[kEmitWarps > 0 ? kEmitWarps : 1];  // minify: completion of an emit warp's block fetch
  sj_mbar_t park_free[kParkFree];  // phase k: every block of element (slot + k * kParkFree) has been emitted, the parked masks may be overwritten
  uint32_t emitted_cnt[kNS];     // blocks of the element emitted so far
  uint32_t emit_next;            // next (element, block) item: element = item / kScanWarps
  uint32_t scan_done;            // 0xFFFFFFFF while the scan warps are running, then the number of elements this CTA scanned
#if SJB200_SCAN4_TRACE
  uint32_t trace[2][kTraceIters][kTracePoints];  // tuning build: SM cycle counter at the phase boundaries of scan warps 0 and 9
  unsigned long long trace_cta[4];               // globaltimer: kernel entry, roles start, scan role done, before exit
#endif
};
constexpr int kSmemBytes4 = int(sizeof(Smem)) + 1024;

// byte offset inside a block -> offset in the 128B-swizzled shared-memory image
SJ_DEV uint32_t swz(uint32_t off) { return off ^ ((off >> 3) & 0x70u); }

// ------------------------------------------------------------------------------------------------ descriptors
// [63:46] epoch  [45:44] status  [43:0] payload
//   aggregate: [38] quote parity of the element, [37:19] outputs if it is entered inside a string, [18:0] ... outside
//   inclusive: [32] in-string after the element, [31:0] outputs of elements [0, i]
SJ_DEV unsigned long long pack_agg(uint32_t epoch, uint32_t par, uint32_t c0, uint32_t c1) {
  return ((unsigned long long)epoch << 46) | ((unsigned long long)kDescAgg << 44) | ((unsigned long long)(par & 1u) << 38) |
         ((unsigned long long)c1 << 19) | c0;
}
SJ_DEV unsigned long long pack_inc(uint32_t epoch, uint32_t s_out, uint32_t count) {
  return ((unsigned long long)epoch << 46) | ((unsigned long long)kDescInc << 44) | ((unsigned long long)(s_out & 1u) << 32) | count;
}

// The effect of a run of elements on (in-string, outputs): p = quote parity, a / b = outputs when entered outside /
// inside a string.  compose(older, newer) is associative; identity = (0,0,0).
struct Eff {
  uint32_t p, a, b;
};
SJ_DEV Eff compose(const Eff &o, const Eff &n) {
  Eff r;
  r.p = o.p ^ n.p;
  r.a = o.a + (o.p ? n.b : n.a);
  r.b = o.b + (o.p ? n.a : n.b);
  return r;
}

// A waiting warp must not spin at full speed: mbarrier.try_wait returns at once, and a busy loop takes issue slots
// from the warps that do the work.  `ns` = back-off between polls.
#ifndef SJB200_SCAN4_POLL_SCALE
#define SJB200_SCAN4_POLL_SCALE 1
#endif
SJ_DEV bool wait_bar(sj_mbar_t *bar, uint32_t parity, const ScanParams &p, unsigned ns) {
  uint32_t spins = 0;
  while (!sj_mbar_try_wait(bar, parity)) {
    if (++spins > kSpinLimit4) {
      sj_atomic_or(p.flags, kFlagInternal);
      return false;
    }
    sj_nanosleep(ns * SJB200_SCAN4_POLL_SCALE);
  }
  return true;
}

// ------------------------------------------------------------------------------------------------ byte helpers
SJ_DEV bool byte_is_scalar(uint32_t b) {
  const bool ws = b == 0x20u || b == 0x09u || b == 0x0Au || b == 0x0Du;
  const bool op = b == 0x2Cu || b == 0x3Au || b == 0x5Bu || b == 0x5Du || b == 0x7Bu || b == 0x7Du || b == 0x0Cu || b == 0x1Au;
  return !(ws || op);
}

// Length of the run of backslashes that ends just before `end` (exclusive), not looking below `floor`.
// *hit_floor: the run reaches `floor`.  Called by a whole warp; the result is uniform.  Rare path (the byte before a
// block is a backslash or a quote): 32 bytes per step, 512 when the run is long and the address allows vector loads.
SJ_DEV uint64_t run_back(const uint8_t *buf, uint64_t end, uint64_t floor, unsigned lane, bool *hit_floor) {
  uint64_t cur = end, total = 0;
  *hit_floor = false;
  uint32_t steps = 0;
  for (;;) {
    if (cur == floor) {
      *hit_floor = true;
      return total;
    }
    if (steps >= 4 && cur - floor >= 512 && ((reinterpret_cast<uintptr_t>(buf) + cur) & 15u) == 0) {
      const sj_u4 v = sj_ldg_u4(buf + cur - 16 * (uint64_t(lane) + 1));
      const bool allbs = (v.x == 0x5C5C5C5Cu) && (v.y == 0x5C5C5C5Cu) && (v.z == 0x5C5C5C5Cu) && (v.w == 0x5C5C5C5Cu);
      const uint32_t m = sj_ballot(!allbs);
      if (m == 0) {
        total += 512;
        cur -= 512;
        continue;
      }
      const uint32_t f = uint32_t(sj_ffs(m) - 1);
      total += 16ull * f;
      cur -= 16ull * f;  // the chunk that stops the run is finished byte by byte below
    }
    const uint64_t avail64 = cur - floor;
    const uint32_t avail = avail64 < 32 ? uint32_t(avail64) : 32u;
    const bool isbs = lane < avail && sj_ldg_u8(buf + cur - 1 - lane) == 0x5Cu;
    const uint32_t m = sj_ballot(!isbs);
    if (m != 0) {
      const uint32_t f = uint32_t(sj_ffs(m) - 1);
      total += f;
      if (f == avail && avail < 32) *hit_floor = true;
      return total;
    }
    total += 32;
    cur -= 32;
    steps++;
  }
}
// ... and the run that starts at `begin`, not looking at or beyond `limit`
SJ_DEV uint64_t run_forward(const uint8_t *buf, uint64_t begin, uint64_t limit, unsigned lane) {
  uint64_t cur = begin, total = 0;
  uint32_t steps = 0;
  for (;;) {
    if (cur >= limit) return total;
    if (steps >= 4 && limit - cur >= 512 && ((reinterpret_cast<uintptr_t>(buf) + cur) & 15u) == 0) {
      const sj_u4 v = sj_ldg_u4(buf + cur + 16 * uint64_t(lane));
      const bool allbs = (v.x == 0x5C5C5C5Cu) && (v.y == 0x5C5C5C5Cu) && (v.z == 0x5C5C5C5Cu) && (v.w == 0x5C5C5C5Cu);
      const uint32_t m = sj_ballot(!allbs);
      if (m == 0) {
        total += 512;
        cur += 512;
        continue;
      }
      const uint32_t f = uint32_t(sj_ffs(m) - 1);
      total += 16ull * f;
      cur += 16ull * f;
    }
    const uint64_t avail64 = limit - cur;
    const uint32_t avail = avail64 < 32 ? uint32_t(avail64) : 32u;
    const bool isbs = lane < avail && sj_ldg_u8(buf + cur + lane) == 0x5Cu;
    const uint32_t m = sj_ballot(!isbs);
    if (m != 0) return total + uint32_t(sj_ffs(m) - 1);
    total += 32;
    cur += 32;
    steps++;
  }
}

// Scanner state entering byte `pos` of the document: bit0 = the byte is escaped (an odd-length backslash run ends at
// pos-1), bit2 = byte pos-1 is a "non-quote scalar" (json_scanner.h L148-149).  Exact for any input: the run is
// followed back as far as it goes, at most to the first byte of this launch, where the launch's carry-in takes over.
// `b1` = byte pos-1.  Warp-uniform.
SJ_DEV uint32_t boundary_state(const ScanParams &p, uint64_t pos, uint64_t launch_start, uint32_t cin_state, uint32_t pw, unsigned lane) {
  if (pos == launch_start) return cin_state & 5u;
  const uint32_t b1 = pw >> 24;
  if (b1 != 0x5Cu && b1 != 0x22u) return byte_is_scalar(b1) ? 4u : 0u;  // the common case: one byte decides
  // a quote's own status depends on the run before it.  Short runs are decided from the four bytes at hand (a quote
  // right before a block boundary is common; going back to global memory for it would cost the warp a round trip to L2)
  const uint32_t b2 = (pw >> 16) & 0xFFu, b3 = (pw >> 8) & 0xFFu, b4 = pw & 0xFFu;
  const bool isq = (b1 == 0x22u);
  uint32_t run = 0xFFFFFFFFu;  // backslashes ending at byte -1 (or at byte -2 when byte -1 is a quote); unknown yet
  if (pos - launch_start >= 4) {
    if (isq) {
      if (b2 != 0x5Cu) run = 0;
      else if (b3 != 0x5Cu) run = 1;
      else if (b4 != 0x5Cu) run = 2;
    } else {
      if (b2 != 0x5Cu) run = 1;
      else if (b3 != 0x5Cu) run = 2;
      else if (b4 != 0x5Cu) run = 3;
    }
  }
  uint32_t odd;
  if (run != 0xFFFFFFFFu) {
    odd = run & 1u;
  } else {
    const uint64_t end = isq ? pos - 1 : pos;
    bool hit = false;
    const uint64_t r = run_back(p.buf, end, launch_start, lane, &hit);
    odd = uint32_t(r + ((hit && (cin_state & 1u)) ? 1u : 0u)) & 1u;
  }
  if (isq) return odd << 2;  // escaped quote = scalar byte; a real quote is not; neither escapes what follows
  return odd | 4u;           // a backslash is a scalar byte
}

// the 4 bytes before document offset `pos` as a little-endian word (byte pos-1 on top)
SJ_DEV uint32_t word_before(const ScanParams &p, uint64_t pos) {
  if (pos == 0) return p.prev_word;
  if (pos >= 4 && ((reinterpret_cast<uintptr_t>(p.buf) + pos) & 3u) == 0) return sj_ldg_u32(p.buf + pos - 4);
  uint32_t w = 0;
  for (int d = 1; d <= 4; d++) {
    const uint32_t b = (pos >= uint64_t(d)) ? sj_ldg_u8(p.buf + pos - d) : ((p.prev_word >> (8 * (4 - d + int(pos)))) & 0xFFu);
    w |= b << (8 * (4 - d));
  }
  return w;
}

// ------------------------------------------------------------------------------------------------ block I/O
// A warp copies one block global -> shared in the swizzled layout, padding with 0x20 past len.  Used for the last
// (partial) block and for buffers TMA cannot address (stage 1 never reads past len: buf_block_reader.h L98-104).
SJ_DEV void fill_block_guarded(uint8_t *T, const ScanParams &p, uint64_t bstart, unsigned lane) {
  const bool aligned = (reinterpret_cast<uintptr_t>(p.buf) & 15u) == 0;
  for (uint32_t c = lane; c < uint32_t(kBlockBytes / 16); c += 32) {
    const uint64_t g = bstart + uint64_t(c) * 16;
    sj_u4 v;
    if (aligned && g + 16 <= p.len) {
      v = sj_ldg_u4(p.buf + g);
    } else {
      uint32_t w[4];
      for (int k = 0; k < 4; k++) {
        uint32_t x = 0;
        for (int b = 0; b < 4; b++) {
          const uint64_t q = g + 4 * k + b;
          const uint32_t byte = (q < p.len) ? sj_ldg_u8(p.buf + q) : 0x20u;
          x |= byte << (8 * b);
        }
        w[k] = x;
      }
      v = sj_make_u4(w[0], w[1], w[2], w[3]);
    }
    *reinterpret_cast<sj_u4 *>(T + swz(c * 16)) = v;
  }
}

SJ_DEV void load_unit(const uint8_t *T, uint32_t off, uint32_t w[8]) {
  const sj_u4 a = *reinterpret_cast<const sj_u4 *>(T + swz(off));
  const sj_u4 b = *reinterpret_cast<const sj_u4 *>(T + swz(off + 16));
  w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
  w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}

// ------------------------------------------------------------------------------------------------ scan one block
// T: the block in shared memory.  pw0: the 4 bytes before the block (only lane 0's copy is used).  e_in / c_in: the two
// locally known state bits entering the block.  Parks the two candidate masks and the lane's exclusive output prefix,
// returns the block summary word (uniform).
// kMin: the minify flavour (json_minifier.h L68-97): no UTF-8 validation, the two candidate masks are the bytes to KEEP
// (everything but whitespace outside strings) among the first `valid_bytes` of the block, the counts are bytes.
template <bool kMin>
SJ_DEV uint32_t scan_block(const uint8_t *T, uint32_t pw0, uint32_t e_in, uint32_t c_in, unsigned lane, const ScanParams &p, sj_u4 *park0,
                           sj_u4 *park1, uint32_t *parkpre, uint32_t valid_bytes) {
  const uint32_t lane_off = lane * 128u;
  uint32_t bs[4], qu[4], op[4], sc[4], cl[4];
  uint32_t uerr = 0;
  if (kMin) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      uint32_t w8[8], pl[8];
      load_unit(T, lane_off + 32u * u, w8);
      transpose32(w8, pl);
      const unit_classes c = classify(pl);
      bs[u] = c.bs; qu[u] = c.qu; op[u] = c.op; sc[u] = c.sc; cl[u] = 0;
    }
  } else {
    // One decision per block instead of one per unit: does any lane hold a byte >= 0x80?  (The lane's row is read
    // twice -- the load pipe has room, the ALU pipe does not.)  An all-ASCII block needs no UTF-8 code at all, any other
    // block runs the check in every unit without the per-unit vote, pending-carry bookkeeping and carry reset.
    uint32_t hi = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const sj_u4 v = *reinterpret_cast<const sj_u4 *>(T + swz(lane_off + 16u * c));
      hi |= v.x | v.y | v.z | v.w;
    }
    if (!sj_any((hi & 0x80808080u) != 0)) {
#pragma unroll
      for (int u = 0; u < 4; u++) {
        uint32_t w8[8], pl[8];
        load_unit(T, lane_off + 32u * u, w8);
        transpose32(w8, pl);
        const unit_classes c = classify(pl);
        bs[u] = c.bs; qu[u] = c.qu; op[u] = c.op; sc[u] = c.sc; cl[u] = c.ctl;
      }
      // only the block before this one can have left a sequence open: it ends in ASCII here, which is an error
      if (lane == 0 && utf8_carry_pending(utf8_carry_from_prev_word(pw0))) uerr = 1u;
    } else {
      const uint32_t pw = (lane == 0) ? pw0 : *reinterpret_cast<const uint32_t *>(T + swz(lane_off - 4));
      utf8_carry uc = utf8_carry_from_prev_word(pw);
#pragma unroll
      for (int u = 0; u < 4; u++) {
        uint32_t w8[8], pl[8];
        load_unit(T, lane_off + 32u * u, w8);
        transpose32(w8, pl);
        const unit_classes c = classify(pl);
        bs[u] = c.bs; qu[u] = c.qu; op[u] = c.op; sc[u] = c.sc; cl[u] = c.ctl;
        uerr |= utf8_check_unit(pl, uc);
      }
    }
  }
  if (!kMin && sj_any(uerr != 0) && lane == 0) sj_atomic_or(p.flags, kFlagUtf8);

  // ---- escapes: which quotes are real (json_escape_scanner.h L96-143, resolved across lanes with one addition)
  uint32_t qr[4];
  {
    const uint32_t bsany = bs[0] | bs[1] | bs[2] | bs[3];
    if (sj_any(bsany != 0)) {
      uint32_t escaped[4];
      const uint32_t esc_out0 = escape_scan<4>(bs, escaped);
#pragma unroll
      for (int u = 0; u < 4; u++) qr[u] = qu[u] & ~escaped[u];
      const bool allbs = (bs[0] & bs[1] & bs[2] & bs[3]) == 0xFFFFFFFFu;
      const uint32_t G = sj_ballot(esc_out0 != 0);
      const uint32_t P = sj_ballot(allbs);
      uint32_t cout_unused;
      const uint32_t carries = escape_carries(G, P, e_in & 1u, &cout_unused) & ~P;
      if (carries != 0) {  // rare: some lane starts right after an unescaped backslash
        const int nlead = leading_backslashes<4>(bs);
        const uint32_t bit = ((carries >> lane) & 1u) ? (1u << (nlead & 31)) : 0u;
#pragma unroll
        for (int u = 0; u < 4; u++) qr[u] ^= qu[u] & (((nlead >> 5) == u) ? bit : 0u);
      }
    } else {
#pragma unroll
      for (int u = 0; u < 4; u++) qr[u] = qu[u];
      if ((e_in & 1u) && lane == 0) qr[0] ^= qu[0] & 1u;
    }
  }

  // ---- strings and pseudo-structurals, for both in-string polarities at the start of the block
  const uint32_t lp = uint32_t(sj_popc(qr[0] ^ qr[1] ^ qr[2] ^ qr[3])) & 1u;
  const uint32_t pb = sj_ballot(lp != 0);
  uint32_t instr = uint32_t(sj_popc(pb & ((1u << lane) - 1u))) & 1u;
  const uint32_t par = uint32_t(sj_popc(pb)) & 1u;
  uint32_t scal_prev = sj_shfl_up((sc[3] & ~qr[3]) >> 31, 1);
  if (lane == 0) scal_prev = c_in & 1u;
  uint32_t prev_nq = scal_prev << 31;
  uint32_t e0[4], e1[4];
  uint32_t hit0 = 0, hit1 = 0, cnt = 0;
#pragma unroll
  for (int u = 0; u < 4; u++) {
    const uint32_t in_string = prefix_xor32(qr[u]) ^ (0u - instr);  // json_string_scanner.h L73
    instr = in_string >> 31;
    if (kMin) {
      const uint32_t ws = ~(op[u] | sc[u]);
      const int nv = int(valid_bytes) - int(lane_off) - 32 * u;       // bytes of this unit that exist (the padding is never output)
      const uint32_t valid = nv >= 32 ? 0xFFFFFFFFu : (nv <= 0 ? 0u : ((1u << nv) - 1u));
      e0[u] = ~(ws & ~in_string) & valid;                             // json_minifier.h L37-40
      e1[u] = ~(ws & in_string) & valid;
      cnt += uint32_t(sj_popc(e0[u])) | (uint32_t(sj_popc(e1[u])) << 16);
      continue;
    }
    const uint32_t nq = sc[u] & ~qr[u];                              // json_scanner.h L148
    const uint32_t follows = shl_in(prev_nq, nq, 1);                 // L149
    prev_nq = nq;
    const uint32_t pm = op[u] | (sc[u] & ~follows);                  // L68-79
    const uint32_t tail0 = in_string ^ qr[u];                        // string tail if the block starts outside a string
    e0[u] = pm & ~tail0;
    e1[u] = pm & tail0;
    hit0 |= cl[u] & in_string;                                       // json_structural_indexer.h L246
    hit1 |= cl[u] & ~in_string;
    cnt += uint32_t(sj_popc(e0[u])) | (uint32_t(sj_popc(e1[u])) << 16);
  }
  uint32_t incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = sj_shfl_up(incl, d);
    if (int(lane) >= d) incl += t;
  }
  const uint32_t total = sj_shfl(incl, 31);
  const unsigned tid = sj_tid();
  park0[tid] = sj_make_u4(e0[0], e0[1], e0[2], e0[3]);
  park1[tid] = sj_make_u4(e1[0], e1[1], e1[2], e1[3]);
  parkpre[tid] = incl - cnt;
  const uint32_t h0 = sj_any(hit0 != 0) ? 1u : 0u, h1 = sj_any(hit1 != 0) ? 1u : 0u;
  return total | (par << 29) | (h0 << 30) | (h1 << 31);
}

// ------------------------------------------------------------------------------------------------ emit one block
// Each lane walks its own four mask words, column by column: every lane runs the trip count of the fullest word of the
// column (uniform), pulls the highest set bit per iteration (one FLO) and stores its position -- descending, so the
// store offset is an immediate of the unrolled loop.
// one step of one word's chain: store the position of the highest remaining bit at q[-k], clear it
#define SJ_EMIT_STEP(m, q, pb)                   \
  {                                              \
    const bool has = (m) != 0;                   \
    const uint32_t h = sj_bfind(m);              \
    (q)--;                                       \
    if (has) *(q) = (pb) + h;                    \
    (m) &= ~(1u << (h & 31u));                   \
  }
SJ_DEV void emit_columns(const sj_u4 ev, uint32_t off, uint32_t pos_lane, uint32_t *dst) {
  // The chains of different words are independent: run them side by side, so that the FLO -> shift -> clear latency of
  // one is covered by the others (a warp that emits is otherwise latency-bound: ~4 dependent instructions per output).
  uint32_t m0 = ev.x, m1 = ev.y, m2 = ev.z, m3 = ev.w;
  const uint32_t c0 = uint32_t(sj_popc(m0)), c1 = uint32_t(sj_popc(m1)), c2 = uint32_t(sj_popc(m2)), c3 = uint32_t(sj_popc(m3));
  uint32_t *q0 = dst + (off + c0);  // one past each word's last output
  uint32_t *q1 = q0 + c1, *q2 = q1 + c2, *q3 = q2 + c3;
  const uint32_t pb0 = pos_lane, pb1 = pos_lane + 32u, pb2 = pos_lane + 64u, pb3 = pos_lane + 96u;
  const uint32_t c01 = c0 > c1 ? c0 : c1, c23 = c2 > c3 ? c2 : c3;
  const uint32_t n = sj_reduce_max(c01 > c23 ? c01 : c23);
#pragma unroll 2
  for (uint32_t k = 0; k < n; k++) {
    SJ_EMIT_STEP(m0, q0, pb0)
    SJ_EMIT_STEP(m1, q1, pb1)
    SJ_EMIT_STEP(m2, q2, pb2)
    SJ_EMIT_STEP(m3, q3, pb3)
  }
}
#undef SJ_EMIT_STEP

// the rare block with more than one output per four bytes: no staging, compact code (kept out of line: the kernel's
// hot loops should stay resident in the instruction cache)
SJ_DEV_NOINLINE void emit_columns_dense(const sj_u4 ev, uint32_t off, uint32_t pos_lane, uint32_t *dst) {
  const uint32_t m4[4] = {ev.x, ev.y, ev.z, ev.w};
  for (int u = 0; u < 4; u++) {
    uint32_t m = m4[u];
    uint32_t *q = dst + off;
    while (m != 0) {
      const uint32_t l = uint32_t(sj_ffs(m)) - 1u;
      *q++ = pos_lane + 32u * uint32_t(u) + l;
      m &= m - 1u;
    }
    off += uint32_t(sj_popc(m4[u]));
  }
}

// emit block `warp` of this CTA's e-th element (resolved).  ev / prew: the lane's parked mask for the polarity the
// block turned out to have and its packed output prefix.  stg: 4 KiB of shared memory nobody else is using.
SJ_DEV void emit_block(Smem *S, const ScanParams &p, uint64_t out_base, uint32_t e, unsigned warp, unsigned lane, const sj_u4 ev, uint32_t prew,
                       uint32_t *stg) {
  const int ns = int(e % kNS);
  const uint32_t sum = S->summary[ns][warp];
  const uint32_t pol = S->res_pol[ns][warp] & 1u;
  const uint32_t total = pol ? ((sum >> 16) & 0x1FFFu) : (sum & 0xFFFFu);
  if (total == 0) return;
  const uint32_t elem = S->ticket[ns];
  const uint32_t off = (prew >> (16 * pol)) & 0xFFFFu;
  const uint32_t pos_lane = p.pos_base + p.tile_begin * uint32_t(kTileBytes) + elem * uint32_t(kElemBytes) + warp * uint32_t(kBlockBytes) + lane * 128u;
  uint32_t *out = p.idx_out + (out_base + S->res_base[ns][warp]);
  if (total + 3 <= kStageWords) {
    // positions go to shared memory (scattered 4-byte global stores cost one L1 wavefront each) and leave as coalesced
    // 16-byte vectors: the staging area starts at the same offset modulo 4 words as the destination, so the aligned
    // groups of the two line up
    const uint32_t a = uint32_t((reinterpret_cast<uintptr_t>(out) >> 2) & 3u);  // out is 4-byte aligned
    sj_syncwarp();
    emit_columns(ev, off, pos_lane, stg + a);
    sj_syncwarp();
    const uint32_t head = (total < ((4u - a) & 3u)) ? total : ((4u - a) & 3u);  // words before the first aligned group
    const uint32_t nvec = (total - head) >> 2;
    const uint32_t tail = total - head - (nvec << 2);
    if (lane < head) out[lane] = stg[a + lane];
    const sj_u4 *sv = reinterpret_cast<const sj_u4 *>(stg + a + head);  // (a + head) % 4 == 0
    sj_u4 *gv = reinterpret_cast<sj_u4 *>(out + head);
    for (uint32_t i = lane; i < nvec; i += 32) gv[i] = sv[i];
    if (lane < tail) out[head + (nvec << 2) + lane] = stg[a + head + (nvec << 2) + lane];
    sj_syncwarp();
  } else {
    emit_columns_dense(ev, off, pos_lane, out);  // > 1 structural per 4 bytes over 4 KiB: straight to global memory
  }
  if (!SJB200_SCAN4_TRACE && p.debug != nullptr && warp == 0 && lane == 0) p.debug[uint64_t(elem) * 8 + 5] = sj_globaltimer();
}

// pipelined mode: the masks wait in shared memory
SJ_DEV void emit_from_smem(Smem *S, const ScanParams &p, uint64_t out_base, uint32_t e, unsigned warp, unsigned lane, uint32_t *stg) {
  const uint32_t pol = S->res_pol[e % kNS][warp] & 1u;
  const unsigned tid = warp * 32 + lane;
  emit_block(S, p, out_base, e, warp, lane, S->park[kGPark > 0 ? 0 : e % kPark][pol][kGPark > 0 ? 0 : tid], S->parkpre[kGPark > 0 ? 0 : e % kPark][kGPark > 0 ? 0 : tid], stg);
}

// emit-warp mode: the masks wait in the scratch ring of ScanParams::park (it stays in L2)
SJ_DEV uint32_t *park_slot(const ScanParams &p, uint32_t e) { return p.park + (size_t(sj_cta()) * kParkRing + (e % uint32_t(kParkRing))) * size_t(kParkSlotWords); }

// ------------------------------------------------------------------------------------------------ minify: emit one block
// kept bytes of a 4-byte word packed to its low end: the PRMT selector (unused positions select a zero byte)
// (computed once per CTA into shared memory: 16 words in 16 banks, any mix of nibbles across the lanes is one access)
SJ_DEV uint32_t compact_entry(uint32_t nib) {
  uint32_t sel = 0, cnt = 0;
  for (uint32_t b = 0; b < 4; b++)
    if ((nib >> b) & 1u) { sel |= b << (4 * cnt); cnt++; }
  for (uint32_t i = cnt; i < 4; i++) sel |= 4u << (4 * i);
  return sel;
}

// minify: start fetching block `warp` of this CTA's e-th element again (two scans old, still in L2) into `slot`.
// Returns true when it comes by TMA (completes `bar`); otherwise emit_minify_block fills the slot itself.
SJ_DEV bool minify_fetch_issue(Smem *S, const sj_tensor_map *tmap, const ScanParams &p, uint32_t e, unsigned warp, unsigned lane, uint8_t *slot, sj_mbar_t *bar,
                               uint64_t launch_start) {
  const uint64_t bstart = launch_start + uint64_t(S->ticket[e % kNS]) * kElemBytes + uint64_t(warp) * kBlockBytes;
  const uint64_t row = bstart / 128;
  const bool by_tma = p.use_tma && (row + kBlockRows <= p.len / 128);
  sj_syncwarp();  // every lane is done with the slot
  if (by_tma && lane == 0) {
    sj_fence_proxy_async();
    sj_mbar_arrive_expect_tx(bar, kBlockBytes);
    sj_tma_load_rows(slot, tmap, bar, uint32_t(row));
  }
  return by_tma;
}

// Block `warp` of this CTA's e-th element (resolved): with its bytes back in `slot` (fetched < 0: not asked for yet;
// 0 / 1: minify_fetch_issue ran and returned that), pull the lane's row into registers, turn the slot into the staging
// area, pack the kept bytes of every word with one PRMT (independent look-ups), then string the packed words together
// -- a shift, an OR and a select per word on the critical path -- storing complete words into the staging area (the
// words at a lane's seams are OR-ed into the zeroed area, lanes share them), and store the block's output as aligned
// 16-byte vectors.  Returns true when the slot's mbarrier completed a phase (the caller tracks parities).
SJ_DEV bool emit_minify_block(Smem *S, const sj_tensor_map *tmap, const ScanParams &p, uint64_t out_base, uint32_t e, unsigned warp, unsigned lane,
                              const sj_u4 kv, uint32_t prew, uint8_t *slot, sj_mbar_t *bar, uint32_t parity, uint64_t launch_start, int fetched = -1) {
  const int ns = int(e % kNS);
  const uint32_t sum = S->summary[ns][warp];
  const uint32_t pol = S->res_pol[ns][warp] & 1u;
  const uint32_t total = pol ? ((sum >> 16) & 0x1FFFu) : (sum & 0xFFFFu);
  if (fetched < 0 && total == 0) return false;
  const uint32_t elem = S->ticket[ns];
  const uint64_t bstart = launch_start + uint64_t(elem) * kElemBytes + uint64_t(warp) * kBlockBytes;
  const bool by_tma = fetched < 0 ? minify_fetch_issue(S, tmap, p, e, warp, lane, slot, bar, launch_start) : fetched != 0;
  if (by_tma) {
    wait_bar(bar, parity, p, 32);
  } else {
    if (total == 0) return false;
    fill_block_guarded(slot, p, bstart, lane);
    sj_syncwarp();
  }
  if (total == 0) return by_tma;
  uint32_t w[32];
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const sj_u4 v = *reinterpret_cast<const sj_u4 *>(slot + swz(lane * 128u + 16u * c));
    w[4 * c] = v.x; w[4 * c + 1] = v.y; w[4 * c + 2] = v.z; w[4 * c + 3] = v.w;
  }
  const uint32_t off = (prew >> (16 * pol)) & 0xFFFFu;  // bytes of the block's output before this lane's
  sj_syncwarp();  // every lane holds its row: the slot becomes the staging area
  // lanes OR into the words at their seams only -- a lane's first word is the previous lane's last one -- so only those
  // are zeroed (complete words are plain stores)
  if (off < uint32_t(kBlockBytes)) *reinterpret_cast<uint32_t *>(slot + swz(off & ~3u)) = 0u;
  if (lane == 31 && total < uint32_t(kBlockBytes)) *reinterpret_cast<uint32_t *>(slot + swz(total & ~3u)) = 0u;
  sj_syncwarp();
  const uint32_t keep[4] = {kv.x, kv.y, kv.z, kv.w};
  // kept bytes per word: the nibble popcounts of the keep masks (0..4 each)
  uint32_t cn[4];
#pragma unroll
  for (int q = 0; q < 4; q++) cn[q] = keep[q] - ((keep[q] >> 1) & 0x77777777u) - ((keep[q] >> 2) & 0x33333333u) - ((keep[q] >> 3) & 0x11111111u);
#pragma unroll
  for (int i = 0; i < 32; i++) w[i] = byte_perm(w[i], 0u, S->compact_lut[(keep[i >> 3] >> (4 * (i & 7))) & 15u]);
  // carry holds sh/8 bytes at its low end (zero above them).  No branches: the first word a lane completes (it may hold
  // bytes of the lanes before it) is kept in a register and OR-ed in after the loop, every other one is a plain store.
  const uint32_t wa0 = off & ~3u;  // byte offset of the first word this lane contributes to
  uint32_t carry = 0, sh = 8u * (off & 3u), wa = wa0, first = 0;
#pragma unroll
  for (int i = 0; i < 32; i++) {
    const uint32_t c8 = (i & 7) == 0 ? (cn[i >> 3] << 3) & 0x38u : (cn[i >> 3] >> (4 * (i & 7) - 3)) & 0x38u;  // 8 * kept bytes of word i
    const uint32_t merged = carry | (w[i] << sh);
    const uint32_t tot = sh + c8;
    const bool done = tot >= 32u;
    const bool is_first = wa == wa0;
    if (done && !is_first) *reinterpret_cast<uint32_t *>(slot + swz(wa)) = merged;
    first = (done && is_first) ? merged : first;
    carry = done ? sj_funnel_l(w[i], 0u, int(sh)) : merged;  // sh = 0: nothing of w[i] is left over
    wa += done ? 4u : 0u;
    sh = tot & 31u;
  }
  if (wa != wa0) sj_atomic_or(reinterpret_cast<uint32_t *>(slot + swz(wa0)), first);
  if (sh) sj_atomic_or(reinterpret_cast<uint32_t *>(slot + swz(wa)), carry);
  sj_syncwarp();
  // ---- copy-out: the destination's 16-byte groups, whatever its alignment.  The staging area is swizzled like a block
  // image (16-byte groups of a 128-byte row XOR-ed with the row number): a lane's output is ~24 words on this kind of
  // input, and with a linear layout the lanes' stores above would hit the same 4 banks 8 at a time.
  uint8_t *dst = p.dst + (out_base + S->res_base[ns][warp]);
  const uint32_t a = uint32_t(reinterpret_cast<uintptr_t>(dst) & 15u);
  const uint32_t head = (total < ((16u - a) & 15u)) ? total : ((16u - a) & 15u);
  const uint32_t nvec = (total - head) >> 4;
  const uint32_t tail = total - head - (nvec << 4);
  if (lane < head) dst[lane] = slot[swz(lane)];
  const uint32_t hw = head >> 2;
  const int hs = int(8u * (head & 3u));
  for (uint32_t i = lane; i < nvec; i += 32) {
    // output vector i = staging bytes [head + 16 i, head + 16 i + 16): inside the aligned groups i and i + 1
    const sj_u4 A = *reinterpret_cast<const sj_u4 *>(slot + swz(16u * i));
    sj_u4 B = A;
    if (head) B = *reinterpret_cast<const sj_u4 *>(slot + swz(16u * i + 16u));  // (exists: head + 16 i + 16 <= total <= 4096)
    uint32_t x0, x1, x2, x3, x4;
    if (hw == 0) { x0 = A.x; x1 = A.y; x2 = A.z; x3 = A.w; x4 = B.x; }
    else if (hw == 1) { x0 = A.y; x1 = A.z; x2 = A.w; x3 = B.x; x4 = B.y; }
    else if (hw == 2) { x0 = A.z; x1 = A.w; x2 = B.x; x3 = B.y; x4 = B.z; }
    else { x0 = A.w; x1 = B.x; x2 = B.y; x3 = B.z; x4 = B.w; }
    *reinterpret_cast<sj_u4 *>(dst + head + 16u * i) = sj_make_u4(sj_funnel_r(x0, x1, hs), sj_funnel_r(x1, x2, hs), sj_funnel_r(x2, x3, hs), sj_funnel_r(x3, x4, hs));
  }
  if (lane < tail) dst[head + (nvec << 4) + lane] = slot[swz(head + (nvec << 4) + lane)];
  sj_syncwarp();
  if (p.debug != nullptr && warp == 0 && lane == 0) p.debug[uint64_t(elem) * 8 + 5] = sj_globaltimer();
  return by_tma;
}

// ------------------------------------------------------------------------------------------------ element summary
// Run by the LAST scan warp to finish an element (so the aggregate is out as early as possible, independent of how far
// the chain warp is with older elements): compose the block summaries for either polarity at the start of the
// element, publish the aggregate in the look-back chain, leave the per-block prefixes for the chain warp.
SJ_DEV void compose_element(Smem *S, const ScanParams &p, int ns, uint32_t t, unsigned lane) {
  // Lane w holds the summary of block w.  Only one bit is order-dependent: the quote parities of the blocks are one
  // ballot word, the polarity entering block w (for an element entered outside a string) is a popcount, and what a block
  // contributes for either polarity of the element is then known per lane -- the element's aggregate is two REDUX sums.
  // It is published at once (it gates every later element of the launch); the per-block prefixes the chain warp needs
  // to post the blocks' output offsets are computed after that.
  const uint32_t r = (lane < uint32_t(kScanWarps)) ? S->summary[ns][lane] : 0u;  // lanes beyond the element: identity
  const uint32_t c0 = r & 0xFFFFu, c1 = (r >> 16) & 0x1FFFu, h0 = (r >> 30) & 1u, h1 = r >> 31;
  const uint32_t P = sj_ballot(((r >> 29) & 1u) != 0);
  const uint32_t s = uint32_t(sj_popc(P & ((1u << lane) - 1u))) & 1u;
  const uint32_t a = s ? c1 : c0, b = s ? c0 : c1;      // this block's outputs when the ELEMENT is entered outside / inside a string
  const uint32_t A = sj_reduce_add(a), B = sj_reduce_add(b);
  const uint32_t HA = sj_any((s ? h1 : h0) != 0) ? 1u : 0u, HB = sj_any((s ? h0 : h1) != 0) ? 1u : 0u;
  const uint32_t par = uint32_t(sj_popc(P)) & 1u;
  if (lane == 0) {
    if (t > 0) sj_st_relaxed_u64(p.count_desc + t, pack_agg(p.epoch, par, A, B));  // element 0 goes straight to inclusive
    S->elem[ns][0] = par;
    S->elem[ns][1] = A;
    S->elem[ns][2] = B;
    S->elem[ns][3] = HA | (HB << 1);
  }
  uint32_t ia = a, ib = b;  // inclusive prefixes over the blocks
#pragma unroll
  for (int d = 1; d < kScanWarps; d <<= 1) {
    const uint32_t xa = sj_shfl_up(ia, d), xb = sj_shfl_up(ib, d);
    if (int(lane) >= d) { ia += xa; ib += xb; }
  }
  if (lane < uint32_t(kScanWarps)) {
    S->pre[ns][0][lane] = (s << 31) | (ia - a);         // entered outside: polarity | outputs before the block
    S->pre[ns][1][lane] = ((s ^ 1u) << 31) | (ib - b);  // entered inside
  }
  sj_syncwarp();
}

// ------------------------------------------------------------------------------------------------ scan warps
SJ_DEV void publish_ticket(Smem *S, uint32_t j, uint32_t value, unsigned lane) {
  if (lane == 0) {
    S->ticket[j % kNS] = value;
    sj_mbar_arrive(&S->ticket_ready[j % kNS]);
  }
  sj_syncwarp();
}

SJ_DEV uint32_t wait_ticket(Smem *S, uint32_t j, const ScanParams &p) {
  if (!wait_bar(&S->ticket_ready[j % kNS], (j / kNS) & 1u, p, 100)) return 0xFFFFFFFFu;
  return S->ticket[j % kNS];
}

// start the load of block `warp` of element `elem` into ring slot r; returns true when it arrives by TMA
SJ_DEV bool issue_load(Smem *S, const sj_tensor_map *tmap, const ScanParams &p, uint32_t elem, unsigned warp, unsigned lane, int r,
                       uint32_t *pw_out, uint64_t scan_limit) {
  const uint64_t bstart = uint64_t(p.tile_begin) * kTileBytes + uint64_t(elem) * kElemBytes + uint64_t(warp) * kBlockBytes;
  const uint64_t row = bstart / 128;
  const bool full = p.use_tma && bstart < scan_limit && (row + kBlockRows <= p.len / 128);
  sj_syncwarp();  // every lane is done with the slot (previous block, emit staging)
  if (lane == 0) {
    if (full) {
      sj_fence_proxy_async();
      sj_mbar_arrive_expect_tx(&S->full[warp][r], kBlockBytes);
      sj_tma_load_rows(S->ring[warp][r], tmap, &S->full[warp][r], uint32_t(row));
    }
    // after the TMA is on its way: the fence above would otherwise sit out this load's round trip to L2
    *pw_out = (bstart < p.len) ? word_before(p, bstart) : 0x20202020u;
  }
  return full;
}

template <int kMode>
SJ_DEV void emit_role(Smem *S, const sj_tensor_map *tmap, const ScanParams &p, const Carry &cin, unsigned lane, uint8_t *stage, sj_mbar_t *fetch_bar,
                      uint32_t fetch_phase);

// kMode: 0 stage 1; 2 minify
template <int kMode>
SJ_DEV void scan_role(Smem *S, const sj_tensor_map *tmap, const ScanParams &p, const Carry &cin, unsigned warp, unsigned lane, uint32_t first_ticket) {
  const uint32_t nelem = elements_of(p);
  const uint64_t launch_start = uint64_t(p.tile_begin) * kTileBytes;
  const uint64_t launch_end = launch_start + uint64_t(p.ntiles) * kTileBytes;
  const uint64_t scan_limit = p.len < launch_end ? p.len : launch_end;  // blocks at or beyond it are not this launch's
  constexpr bool kMin = (kMode == 2);
  const uint64_t out_base = cin.count;
  uint32_t full_phase = 0;
  uint32_t pw_cur = 0x20202020u, pw_next = 0x20202020u;
  bool tma_cur = false, tma_next = false;
  // Tickets must not depend on the chain warp's progress (it may sit in a look-back while the scan warps run ahead),
  // and nobody should wait for a ticket at the top of an iteration (with the ticket published after warp 0's scan,
  // every other warp waited for it in every iteration): the ticket of element j + 2 is
  // drawn and published at the top of iteration j, it is needed at the top of iteration j + 1.
  // Tickets should be scanned in roughly the order they were taken (every element waits for ALL lower tickets): at
  // start-up the second ticket is therefore taken only once the first block has arrived, when every CTA of the launch
  // has drawn its first one.
  if (warp == 0) publish_ticket(S, 0, first_ticket, lane);  // (thread 0 drew it at the top of the kernel)
  uint32_t t = wait_ticket(S, 0, p);
  if (t < nelem) tma_cur = issue_load(S, tmap, p, t, warp, lane, 0, &pw_cur, scan_limit);
  if (warp == 0) {
    if (tma_cur) wait_bar(&S->full[0][0], 0u, p, 32);
    uint32_t a1 = 0;
    if (lane == 0) a1 = sj_atomic_add(p.ticket, 1u);
    publish_ticket(S, 1, a1, lane);
  }
  uint32_t ne = 0;  // this CTA's next element to emit (elements are emitted in order)
  uint32_t j = 0;
  constexpr bool kEmitW = (kEmitWarps > 0);  // the emit warps take the blocks from here: this warp only scans
  for (;; j++) {
    if (t >= nelem) break;
    const int r = int(j & 1u);
    SJ_TRACE4(0);
    const uint32_t tn = wait_ticket(S, j + 1, p);
    if (warp == (j % uint32_t(kScanWarps))) {
      // ticket duty rotates: this warp draws the CTA's element j + 2 and waits for the atomic's round trip
      // before it goes on; the others need that ticket one iteration from now.  (A ticket is scanned two iterations after
      // it was drawn -- every element of the launch waits for ALL lower tickets, so tickets should not be held longer
      // than the TMA pipeline needs -- and no warp is always the one that pays for the round trip.)  Drawn only after
      // ticket j + 1 has been seen: a CTA's tickets must increase with j (the loops stop at the first one beyond the end).
      uint32_t a = 0;
      if (lane == 0) a = sj_atomic_add(p.ticket, 1u);
      publish_ticket(S, j + 2, a, lane);
    }
    SJ_TRACE4(1);
    if (tn < nelem) tma_next = issue_load(S, tmap, p, tn, warp, lane, r ^ 1, &pw_next, scan_limit);
    SJ_TRACE4(2);
    uint8_t *T = S->ring[warp][r];
    const uint64_t bstart = launch_start + uint64_t(t) * kElemBytes + uint64_t(warp) * kBlockBytes;
    if (!SJB200_SCAN4_TRACE && p.debug != nullptr && warp == 0 && lane == 0) {
      p.debug[uint64_t(t) * 8 + 0] = sj_globaltimer();
      p.debug[uint64_t(t) * 8 + 7] = ((unsigned long long)sj_smid() << 48) | ((unsigned long long)sj_cta() << 32) | j;
    }
    uint32_t summary = 0;
    if (bstart < scan_limit) {
      if (tma_cur) {
        wait_bar(&S->full[warp][r], (full_phase >> r) & 1u, p, 32);
        full_phase ^= 1u << r;
      } else {
        fill_block_guarded(T, p, bstart, lane);
        sj_syncwarp();
      }
      SJ_TRACE4(3);
      const uint32_t pw0 = sj_shfl(pw_cur, 0);
      const uint32_t st = boundary_state(p, bstart, launch_start, cin.state, pw0, lane);
      SJ_TRACE4(4);
      {
        // the parked masks of element j - kParkFree must have been emitted before this element's take their place
        if (kEmitW && j >= uint32_t(kParkFree)) wait_bar(&S->park_free[j % kParkFree], ((j / kParkFree) - 1u) & 1u, p, 64);
        const uint64_t left = p.len - bstart;  // > 0: bytes of the block that exist
        const uint32_t valid = left < uint64_t(kBlockBytes) ? uint32_t(left) : uint32_t(kBlockBytes);
        if (kEmitW && kGPark > 0) {
          uint32_t *slot = park_slot(p, j);
          summary = scan_block<kMin>(T, pw0, st & 1u, (st >> 2) & 1u, lane, p, reinterpret_cast<sj_u4 *>(slot), reinterpret_cast<sj_u4 *>(slot) + kScanWarps * 32,
                                     slot + 2 * kScanWarps * 32 * 4, valid);
        } else {
          summary = scan_block<kMin>(T, pw0, st & 1u, (st >> 2) & 1u, lane, p, S->park[j % kPark][0], S->park[j % kPark][1], S->parkpre[j % kPark], valid);
        }
      }
    }
    if (!SJB200_SCAN4_TRACE && p.debug != nullptr && warp == 0 && lane == 0) p.debug[uint64_t(t) * 8 + 1] = sj_globaltimer();
    // minify: the slot just scanned is free -- ask for the block that is emitted below now, the fetch (L2) runs while the
    // element is composed and resolved
    int fetched = -1;
    if (kMin && !kEmitW && j >= uint32_t(kLag)) fetched = minify_fetch_issue(S, tmap, p, ne, warp, lane, T, &S->full[warp][r], launch_start) ? 1 : 0;
    SJ_TRACE4(5);
    {
      const int ns = int(j % kNS);
      uint32_t last = 0;
      if (lane == 0) {
        S->summary[ns][warp] = summary;
        sj_fence_block();
        last = (sj_atomic_add(&S->arrived[ns], 1u) == uint32_t(kScanWarps - 1)) ? 1u : 0u;
      }
      if (sj_shfl(last, 0)) {
        sj_fence_block();
        if (!SJB200_SCAN4_TRACE && p.debug != nullptr && lane == 0) p.debug[uint64_t(t) * 8 + 3] = sj_globaltimer();
        compose_element(S, p, ns, t, lane);
        if (lane == 0) {
          S->arrived[ns] = 0;
          sj_mbar_arrive(&S->scanned[ns]);
        }
      }
    }
    SJ_TRACE4(6);
    SJ_TRACE4(7);
    if (!kEmitW && j >= uint32_t(kLag)) {  // pipelined: the chain warp has had kLag scans' time to resolve this one
      wait_bar(&S->resolved[ne % kNS], (ne / kNS) & 1u, p, 64);
      SJ_TRACE4(8);
      if (!SJB200_SCAN4_TRACE && p.debug != nullptr && warp == 0 && lane == 0) p.debug[uint64_t(S->ticket[ne % kNS]) * 8 + 2] = sj_globaltimer();
      if (kMin) {
        const uint32_t pol = S->res_pol[ne % kNS][warp] & 1u;
        if (emit_minify_block(S, tmap, p, out_base, ne, warp, lane, S->park[kGPark > 0 ? 0 : ne % kPark][pol][kGPark > 0 ? 0 : warp * 32 + lane], S->parkpre[kGPark > 0 ? 0 : ne % kPark][kGPark > 0 ? 0 : warp * 32 + lane], T,
                              &S->full[warp][r], (full_phase >> r) & 1u, launch_start, fetched))
          full_phase ^= 1u << r;
      } else {
        emit_from_smem(S, p, out_base, ne, warp, lane, reinterpret_cast<uint32_t *>(T));
      }
      ne++;
      SJ_TRACE4(9);
    }
    t = tn;
    tma_cur = tma_next;
    pw_cur = pw_next;
  }
  // drain: what this CTA scanned and has not emitted yet (no load is in flight: both ring slots are free)
  if (kEmitW) {
    if (warp == 0 && lane == 0) sj_st_release_u32(&S->scan_done, j);  // the emit warps stop after element j - 1
    sj_syncwarp();
    // nothing left to scan: help with what is left to emit (both ring slots are free: slot 0 is the staging area)
    emit_role<kMode>(S, tmap, p, cin, lane, S->ring[warp][0], &S->full[warp][0], full_phase & 1u);
  } else {
    while (ne < j) {
      wait_bar(&S->resolved[ne % kNS], (ne / kNS) & 1u, p, 64);
      if (kMin) {
        const uint32_t pol = S->res_pol[ne % kNS][warp] & 1u;
        if (emit_minify_block(S, tmap, p, out_base, ne, warp, lane, S->park[kGPark > 0 ? 0 : ne % kPark][pol][kGPark > 0 ? 0 : warp * 32 + lane], S->parkpre[kGPark > 0 ? 0 : ne % kPark][kGPark > 0 ? 0 : warp * 32 + lane],
                              S->ring[warp][0], &S->full[warp][0], full_phase & 1u, launch_start))
          full_phase ^= 1u;
      } else {
        emit_from_smem(S, p, out_base, ne, warp, lane, reinterpret_cast<uint32_t *>(S->ring[warp][0]));
      }
      ne++;
    }
  }
}

// ------------------------------------------------------------------------------------------------ emit warps
// Items are (element, block) pairs in the order the CTA scanned them; a warp takes the next item, waits until the
// element is resolved, emits the block exactly as the scanning warp would have (same parked words, same staging scheme,
// its own staging area), and reports it.  The last block of an element frees the element's parked masks.
template <int kMode>
SJ_DEV void emit_role(Smem *S, const sj_tensor_map *tmap, const ScanParams &p, const Carry &cin, unsigned lane, uint8_t *stage, sj_mbar_t *fetch_bar,
                      uint32_t fetch_phase) {  // stage: this warp's 4 KiB staging area; minify fetches blocks into it through fetch_bar (next parity: fetch_phase)
  const uint64_t out_base = cin.count;
  const uint64_t launch_start = uint64_t(p.tile_begin) * kTileBytes;
  uint32_t *stg = reinterpret_cast<uint32_t *>(stage);
  for (;;) {
    uint32_t q = 0;
    if (lane == 0) q = sj_atomic_add(&S->emit_next, 1u);
    q = sj_shfl(q, 0);
    const uint32_t e = q / uint32_t(kScanWarps), b = q % uint32_t(kScanWarps);
    // until element e is resolved -- or the scan warps report that this CTA never drew an element e
    uint32_t spins = 0;
    for (;;) {
      if (sj_mbar_try_wait(&S->resolved[e % kNS], (e / kNS) & 1u)) break;
      const uint32_t done = sj_ld_acquire_u32(&S->scan_done);
      if (done != 0xFFFFFFFFu && e >= done) return;
      if (++spins > kSpinLimit4) {
        sj_atomic_or(p.flags, kFlagInternal);
        return;
      }
      sj_nanosleep(32);
    }
    const uint32_t pol = S->res_pol[e % kNS][b] & 1u;
    const unsigned tid = b * 32u + lane;
    sj_u4 ev;
    uint32_t prew;
    if (kGPark > 0) {
      const uint32_t *slot = park_slot(p, e);
      ev = sj_ld_u4(slot + (pol * kScanWarps * 32 + tid) * 4);
      prew = sj_ld_u32(slot + 2 * kScanWarps * 32 * 4 + tid);
    } else {
      ev = S->park[kGPark > 0 ? 0 : e % kPark][pol][kGPark > 0 ? 0 : tid];
      prew = S->parkpre[kGPark > 0 ? 0 : e % kPark][kGPark > 0 ? 0 : tid];
    }
    if (kMode == 2) {
      if (emit_minify_block(S, tmap, p, out_base, e, b, lane, ev, prew, stage, fetch_bar, fetch_phase, launch_start)) fetch_phase ^= 1u;
    } else {
      emit_block(S, p, out_base, e, b, lane, ev, prew, stg);
    }
    sj_syncwarp();
    if (lane == 0) {
      sj_fence_block();
      if (sj_atomic_add(&S->emitted_cnt[e % kNS], 1u) == uint32_t(kScanWarps - 1)) {
        S->emitted_cnt[e % kNS] = 0;
        sj_mbar_arrive(&S->park_free[e % kParkFree]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ chain warp

// Decoupled look-back: in-string state and output count entering element t (t >= 1).
// A window is 32*kLookK descriptors, laid out k-major: load k of lane L is the descriptor at distance 32k + L behind
// t-1, so every load instruction of the warp reads 256 contiguous bytes (all CTAs poll the same few cache lines of L2:
// with a lane-major layout every poll was ~200 line requests per warp and the chain warps queued behind one another).
// The window is complete when everything newer than the nearest inclusive prefix has arrived.  Folding uses the fact
// that only one bit is order-dependent: the quote parities of a group of 32 elements are one ballot word, an element's
// polarity relative to the oldest element of the window is a popcount, and the counts are then plain sums.
SJ_DEV void look_back(const ScanParams &p, uint32_t t, unsigned lane, uint32_t *s_in, uint32_t *base) {
  Eff acc;
  acc.p = 0; acc.a = 0; acc.b = 0;
  int64_t newest = int64_t(t) - 1;
  const uint32_t key_agg = (p.epoch << 2) | kDescAgg;  // bits [63:44] of a descriptor of this launch: key_agg or key_agg + 1
  for (;;) {
    const int64_t first = newest - int64_t(lane);  // my k-th descriptor is first - 32k
    unsigned long long d[kLookK];
    uint32_t pend = 0;  // bit k: wanted and not yet arrived
#pragma unroll
    for (int k = 0; k < kLookK; k++) {
      d[k] = 0;
      if (first - 32 * k >= 0) pend |= 1u << k;
    }
    const uint32_t want = pend;
    uint32_t inc_dist = 0xFFFFFFFFu, needed = (1u << kLookK) - 1u;
    uint32_t spins = 0;
    for (;;) {
      // one poll: independent predicated loads straight into d[k] (a word that has not arrived is simply loaded again
      // by the next poll), then three independent instructions per word
      const uint32_t todo = pend;
#pragma unroll
      for (int k = 0; k < kLookK; k++)
        if (todo & (1u << k)) d[k] = sj_ld_relaxed_u64(p.count_desc + (first - 32 * k));
      uint32_t okm = 0, incm = 0;
#pragma unroll
      for (int k = 0; k < kLookK; k++) {
        const uint32_t rel = uint32_t(d[k] >> 44) - key_agg;  // 0: aggregate, 1: inclusive, anything else: not this launch's
        if (rel <= 1u) okm |= 1u << k;
        if (rel == 1u) incm |= 1u << k;
      }
      pend &= ~okm;
      incm &= want;
      // nearest inclusive prefix: for one lane a smaller k is nearer
      const uint32_t my_dist = incm ? uint32_t(sj_ffs(incm) - 1) * 32u + lane : 0xFFFFFFFFu;
      inc_dist = sj_reduce_min(my_dist);
      if (inc_dist != 0xFFFFFFFFu) {  // needed: distance < inc_dist  <=>  k < ceil((inc_dist - lane) / 32)
        const uint32_t nk = (inc_dist > lane) ? (inc_dist - lane + 31u) / 32u : 0u;
        needed = (1u << nk) - 1u;
      }
      if (!sj_any((pend & needed) != 0)) break;
      if (++spins > kSpinLimit4) {  // never expected: report, and finish with what there is
        sj_atomic_or(p.flags, kFlagInternal);
        break;
      }
    }
    // ---- fold the aggregates newer than the inclusive prefix
    const uint32_t use = want & ~pend & needed;
    uint32_t bal[kLookK];
#pragma unroll
    for (int k = 0; k < kLookK; k++) bal[k] = sj_ballot(((use >> k) & 1u) && ((uint32_t(d[k] >> 38) & 1u) != 0));
    uint32_t older = 0;  // parity of everything older than group k (uniform)
    uint32_t sa = 0, sb = 0;
#pragma unroll
    for (int k = kLookK - 1; k >= 0; k--) {
      const uint32_t rel = (uint32_t(sj_popc((bal[k] >> lane) >> 1)) ^ older) & 1u;  // my element's polarity relative to the window's oldest
      if ((use >> k) & 1u) {
        const uint32_t a = uint32_t(d[k]) & 0x7FFFFu, b = uint32_t(d[k] >> 19) & 0x7FFFFu;
        sa += rel ? b : a;
        sb += rel ? a : b;
      }
      older ^= uint32_t(sj_popc(bal[k])) & 1u;
    }
    Eff win;
    win.p = older;
    win.a = sj_reduce_add(sa);
    win.b = sj_reduce_add(sb);
    acc = compose(win, acc);
    if (inc_dist != 0xFFFFFFFFu) {
      const uint32_t ik = inc_dist >> 5, il = inc_dist & 31u;
      uint32_t sk = 0, ck = 0;
#pragma unroll
      for (int k = 0; k < kLookK; k++)
        if (uint32_t(k) == ik) { sk = uint32_t(d[k] >> 32) & 1u; ck = uint32_t(d[k]); }
      sk = sj_shfl(sk, int(il));
      ck = sj_shfl(ck, int(il));
      *s_in = sk ^ acc.p;
      *base = ck + (sk ? acc.b : acc.a);
      return;
    }
    newest -= 32 * kLookK;
    if (newest < 0) {  // cannot happen (element 0 always publishes an inclusive prefix); never loop forever
      sj_atomic_or(p.flags, kFlagInternal);
      *s_in = acc.p;
      *base = acc.a;
      return;
    }
  }
}

// The launch is over: total count, outgoing scanner state, the 6-bit carry transducer of everything it scanned
// (multi-GPU shards fold these: SURVEY.md 8e), sentinels, end-of-input UTF-8 rule.
SJ_DEV void finalize_launch(const ScanParams &p, const Carry &cin, uint32_t s_out, uint64_t count_total, unsigned lane) {
  const uint64_t launch_start = uint64_t(p.tile_begin) * kTileBytes;
  const uint64_t end_scanned = launch_start + uint64_t(p.ntiles) * kTileBytes;
  const uint64_t end_real = p.len < end_scanned ? p.len : end_scanned;
  // state after the last real byte, for the carry-in this launch actually had
  const uint32_t st = boundary_state(p, end_real, launch_start, cin.state, word_before(p, end_real), lane);
  const uint32_t e_a = st & 1u, c_a = (st >> 2) & 1u, par_a = (s_out ^ (cin.state >> 1)) & 1u;
  // ... and for the opposite incoming escape: it can only toggle the first byte that is not a backslash
  const uint64_t nlead = run_forward(p.buf, launch_start, end_real, lane);
  uint32_t e_o = e_a, c_o = c_a, par_o = par_a;
  if (launch_start + nlead >= end_real) {
    e_o ^= 1u;  // nothing but backslashes: the carry goes straight through
  } else if (sj_ldg_u8(p.buf + launch_start + nlead) == 0x22u) {
    par_o ^= 1u;
    if (launch_start + nlead == end_real - 1) c_o ^= 1u;
  }
  const uint32_t ein = cin.state & 1u;
  const uint32_t T0 = ein ? (e_o | (par_o << 1) | (c_o << 2)) : (e_a | (par_a << 1) | (c_a << 2));
  const uint32_t T1 = ein ? (e_a | (par_a << 1) | (c_a << 2)) : (e_o | (par_o << 1) | (c_o << 2));
  if (lane == 0) {
    p.carry_out->count = count_total;
    p.carry_out->state = e_a | (s_out << 1) | (c_a << 2);
    p.carry_out->ttable = T0 | (T1 << 3);
    if (p.carry_out_host != nullptr) {
      p.carry_out_host->count = count_total;
      p.carry_out_host->state = e_a | (s_out << 1) | (c_a << 2);
      p.carry_out_host->ttable = T0 | (T1 << 3);
    }
    if (p.write_sentinels) {  // json_structural_indexer.h L284-286
      uint32_t *tail = p.idx_out + count_total;
      tail[0] = uint32_t(p.len);
      tail[1] = uint32_t(p.len);
      tail[2] = 0;
    }
    if (p.check_eof) {  // utf8_checker::check_eof (utf8_lookup4_algorithm.h L167-171)
      const uint32_t tw = word_before(p, p.len);
      if (utf8_carry_pending(utf8_carry_from_prev_word(tw))) sj_atomic_or(p.flags, kFlagUtf8);
    }
  }
}

SJ_DEV void chain_role(Smem *S, const ScanParams &p, const Carry &cin, unsigned lane, unsigned c) {
  const uint32_t nelem = elements_of(p);
  for (uint32_t j = c;; j += uint32_t(kChainWarps)) {
    const int ns = int(j % kNS);
    const uint32_t t = wait_ticket(S, j, p);
    if (t >= nelem) break;
    uint32_t s_in = (cin.state >> 1) & 1u, base = 0;
    // The look-back needs the elements BEFORE t, not t itself: it runs while this CTA is still scanning t, so that the
    // element is resolved as soon as its own summary is there (with the look-back after the scan, an element waited
    // after the last of its predecessors had been scanned for the pick-up, the poll round trips and the fold).
    if (t > 0) look_back(p, t, lane, &s_in, &base);
    wait_bar(&S->scanned[ns], (j / kNS) & 1u, p, 64);
    if (!SJB200_SCAN4_TRACE && p.debug != nullptr && lane == 0) p.debug[uint64_t(t) * 8 + 6] = sj_globaltimer();
    const uint32_t par = S->elem[ns][0], b0 = S->elem[ns][1], b1 = S->elem[ns][2], hits = S->elem[ns][3];
    const uint32_t mine_total = s_in ? b1 : b0;
    const uint32_t s_out = s_in ^ par;
    if (lane == 0) sj_st_relaxed_u64(p.count_desc + t, pack_inc(p.epoch, s_out, base + mine_total));
    if (lane < uint32_t(kScanWarps)) {
      const uint32_t pk = S->pre[ns][s_in][lane];
      S->res_pol[ns][lane] = pk >> 31;
      S->res_base[ns][lane] = base + (pk & 0x7FFFFFFFu);
    }
    const uint32_t hit0 = hits & 1u, hit1 = (hits >> 1) & 1u;
    if (lane == 0 && (s_in ? hit1 : hit0)) sj_atomic_or(p.flags, kFlagCtl);
    sj_syncwarp();
    if (lane == 0) sj_mbar_arrive(&S->resolved[ns]);
    if (!SJB200_SCAN4_TRACE && p.debug != nullptr && lane == 0) p.debug[uint64_t(t) * 8 + 4] = sj_globaltimer();
    if (t == nelem - 1) finalize_launch(p, cin, s_out, cin.count + base + mine_total, lane);
  }
}

// ------------------------------------------------------------------------------------------------ the kernel body
template <int kMode>
SJ_DEV void scan4_body(const sj_tensor_map *tmap, const ScanParams &p, uint8_t *smem_raw, uint32_t smem_raw_addr) {
  // 1 KiB alignment for the 128B swizzle, computed on the shared-space address so the pointer keeps its address space
  Smem *S = reinterpret_cast<Smem *>(smem_raw + ((1024u - (smem_raw_addr & 1023u)) & 1023u));
  const unsigned tid = sj_tid(), lane = tid & 31u, warp = tid >> 5;
#if SJB200_SCAN4_TRACE
  if (tid == 0) {
    S->trace_cta[0] = sj_globaltimer();
    for (int a = 0; a < 2; a++)
      for (int b = 0; b < kTraceIters; b++)
        for (int cc = 0; cc < kTracePoints; cc++) S->trace[a][b][cc] = 0;
  }
#endif
  // the CTA's first ticket: the atomic's round trip overlaps the set-up below
  uint32_t first_ticket = 0;
  if (tid == 0) first_ticket = sj_atomic_add(p.ticket, 1u);
  Carry cin;
  cin.count = 0; cin.state = 0; cin.ttable = 0; cin.flags = 0; cin.reserved = 0;
  if (p.carry_in != nullptr) cin = *p.carry_in;
  // ~140 mbarriers: one thread each (a single thread initialising them all is slow)
  if (tid < unsigned(kNS)) {
    sj_mbar_init(&S->ticket_ready[tid], 1);
    sj_mbar_init(&S->scanned[tid], 1);
    sj_mbar_init(&S->resolved[tid], 1);
    S->arrived[tid] = 0;
    S->emitted_cnt[tid] = 0;
  } else if (tid < unsigned(kNS + 2 * kScanWarps)) {
    const unsigned k = tid - unsigned(kNS);
    sj_mbar_init(&S->full[k >> 1][k & 1u], 1);
  } else if (tid < unsigned(kNS + 2 * kScanWarps + kParkFree)) {
    sj_mbar_init(&S->park_free[tid - unsigned(kNS + 2 * kScanWarps)], 1);
  } else if (tid < unsigned(kNS + 2 * kScanWarps + kParkFree + (kEmitWarps > 0 ? kEmitWarps : 1))) {
    sj_mbar_init(&S->efull[tid - unsigned(kNS + 2 * kScanWarps + kParkFree)], 1);
  }
  if (tid == 0) {
    S->emit_next = 0;
    S->scan_done = 0xFFFFFFFFu;
  }
  if (tid < unsigned(kNS + 2 * kScanWarps + kParkFree + (kEmitWarps > 0 ? kEmitWarps : 1))) sj_fence_mbar_init();
  if (kMode == 2 && tid < 16) S->compact_lut[tid] = compact_entry(tid);
  sj_syncthreads();
#if SJB200_SCAN4_TRACE
  if (tid == 0) S->trace_cta[1] = sj_globaltimer();
#endif
  if (warp < unsigned(kScanWarps)) scan_role<kMode>(S, tmap, p, cin, warp, lane, first_ticket);
  else if (warp < unsigned(kScanWarps + kChainWarps)) chain_role(S, p, cin, lane, warp - unsigned(kScanWarps));
  else emit_role<kMode>(S, tmap, p, cin, lane, S->estage[warp - unsigned(kScanWarps + kChainWarps)], &S->efull[warp - unsigned(kScanWarps + kChainWarps)], 0u);
#if SJB200_SCAN4_TRACE
  if (tid == 0) S->trace_cta[2] = sj_globaltimer();
#endif
  // last CTA out resets the ticket for the next launch on this context and hands the flags over
  sj_syncthreads();
#if SJB200_SCAN4_TRACE
  if (tid == 0 && p.debug != nullptr) {  // rows: [cta][0] = 4 CTA times + smid; [cta][1 + a * kTraceIters + b] = the 12 points of warp a, iteration b
    unsigned long long *row = p.debug + size_t(sj_cta()) * (1 + 2 * kTraceIters) * 8;
    row[0] = S->trace_cta[0]; row[1] = S->trace_cta[1]; row[2] = S->trace_cta[2]; row[3] = sj_globaltimer(); row[4] = sj_smid();
    for (int a = 0; a < 2; a++)
      for (int b = 0; b < kTraceIters; b++) {
        unsigned long long *q = row + size_t(1 + a * kTraceIters + b) * 8;
        for (int cc = 0; cc < 6; cc++) q[cc] = (unsigned long long)S->trace[a][b][2 * cc] | ((unsigned long long)S->trace[a][b][2 * cc + 1] << 32);
      }
  }
#endif
  if (tid == 0) {
    sj_threadfence();
    const uint32_t done = sj_atomic_add(p.ticket + 1, 1u);
    if (done == sj_nctas() - 1) {
      p.ticket[0] = 0;
      p.ticket[1] = 0;
      p.ticket[2] = 0;
      const uint32_t fl = sj_atomic_exch(p.flags, 0u);
      p.carry_out->flags = fl;
      if (p.carry_out_host != nullptr) p.carry_out_host->flags = fl;
      if (p.xchg_nranks != 0) {
        // the exchange step of a sharded scan, fused: this launch's record goes straight into every rank's window
        // (finalize_launch's stores are visible here: its CTA fenced before it counted itself out)
        const volatile Carry *co = p.carry_out;
        const unsigned long long w0 = xchg_word0(p.xchg_seq, co->count), w1 = xchg_word1(p.xchg_seq, co->state, co->ttable, fl);
        for (uint32_t r = 0; r < p.xchg_nranks; r++) {
          unsigned long long *rec = p.xchg_peer[r] + (size_t(p.xchg_slot) * kMaxRanks + p.xchg_rank) * 2;
          sj_st_sys_u64(rec, w0);
          sj_st_sys_u64(rec + 1, w1);
        }
      }
      sj_threadfence();
    }
  }
}

}  // namespace scan4
}  // namespace sjb200
