// sjb200_tape.cu -- stage-2-lite on the device (SURVEY.md section 8(f) row 4): what the reference's stage 2 decides about
// every token FROM ITS BYTES ALONE, for all structurals of a stage-1 result at once.
//
// What it replaces in the reference (CPU, one token after the other while the tape is built):
//   json_iterator::visit_primitive            src/generic/stage2/json_iterator.h L338-360   (dispatch on the first byte)
//   tape_builder::visit_string -> parse_string  src/generic/stage2/tape_builder.h L186-205, stringparsing.h L146-190
//     handle_unicode_codepoint L55-98, jsoncharutils::codepoint_to_utf8 include/simdjson/generic/jsoncharutils.h L37-62
//     string_buf record [uint32 length][bytes][0], tape payload = its offset (tape_builder.h on_start_string / on_end_string)
//   numberparsing::parse_number               include/simdjson/generic/numberparsing.h L860-961 (grammar, int64 / uint64, value)
//   atomparsing::is_valid_{true,false,null}_atom  include/simdjson/generic/atomparsing.h L45-95
// Not here: the nesting grammar (commas, colons, matching brackets -- the sequential part of stage 2) and the
// conversion of floats (a float is recognised and delimited, type 'd'; the reference also rejects floats whose VALUE is
// infinite, numberparsing.h L765-813).
//
// Three launches, no host round trip between them; a tile = kTokThreads consecutive structurals, one per thread:
//   A  token_scan_kernel   type and payload of every token (a string's payload is its unescaped length for now),
//                          per-tile sums of the string_buf bytes
//   S  tile_scan_kernel    exclusive scan of the tile sums (one CTA), totals; in a sharded pass (sjb200_comm) also the
//                          shard's record and summary, stored into every rank's exchange window
//   B  string_write_kernel every string's record offset (tile offset + CTA scan), the record itself (second walk over
//                          the string, now writing), payload = offset
// Data movement: the bytes a tile's tokens live in are one contiguous span of the document (from its first structural to
// the first structural of the next tile, ~11 bytes per structural): the CTA stages it in shared memory with coalesced
// 16-byte loads and the threads walk their tokens there (whatever does not fit, or lies outside, is read from global
// memory: WindowSrc).  Likewise a tile's string records are one contiguous span of the string buffer: they are composed
// in shared memory at the destination's 16-byte phase and leave as coalesced vectors.  (Per-thread byte loads / stores
// straight to global memory cost one L1 wavefront per touched line and lane: an order of magnitude more.)
// The string buffer comes out byte-identical to dom::document::string_buf of the reference for the same document.
#include <cuda_runtime.h>
#include <stdint.h>

#include "sjb200_common.h"
#include "sjb200_tape.h"
#include "sjb200_tokens.cuh"
#include "sjb200_tokens_warp.cuh"

namespace sjb200 {

namespace {

constexpr int kTokThreads = 256;           // structurals per tile, one per thread (4 CTAs per SM: a CTA's warps finish at different
                                           // times and wait at its barriers -- 2 CTAs of 512 left a third of the issue slots idle)
constexpr uint32_t kWinBytes = 12 * 1024;  // staged input span per tile (~2.8 KB on average)
constexpr uint32_t kOutBytes = 12 * 1024;  // staged string records per tile (B only)
constexpr uint64_t kLaneBudget = 96;       // a lane walks at most this many bytes of a string itself; longer strings go to the warp
constexpr unsigned long long kLongFlag = 1ull << 63;  // payload between A and B: the string was measured by the warp, B copies it the same way

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long *sh) {
  for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, d);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long s = 0;
  for (int w = 0; w < kTokThreads / 32; w++) s += sh[w];
  return s;
}

// Stage the span of the document this tile's tokens live in: win[k] = buf[lo + k] for k < span (span <= kWinBytes).
// lo is rounded down so that buf + lo is 16-byte aligned (whole vectors, never beyond len: the last bytes come one by one).
// The span reaches kWinMargin bytes past the next tile's first structural (what a token of this tile may look at:
// tok::FastWin); *fast: all of that fits, and win is padded with spaces past the end of the document.
constexpr uint32_t kWinMargin = 16;
__device__ tok::WindowSrc stage_window(const uint8_t *buf, uint64_t len, const uint32_t *idx, uint32_t n, uint32_t i0, uint8_t *win, bool *fast) {
  tok::WindowSrc src;
  src.buf = buf; src.len = len; src.win = win;
  const uint64_t first = idx[i0];
  const uint64_t next = (uint64_t(i0) + kTokThreads < n) ? uint64_t(idx[i0 + kTokThreads]) : len;
  const uint64_t mis = (reinterpret_cast<uintptr_t>(buf) + first) & 15u;
  const uint64_t lo = first >= mis ? first - mis : first;  // (first < mis: an unaligned buffer's first bytes; byte loads below)
  uint64_t span = next + kWinMargin - lo;
  *fast = span + kWinMargin <= kWinBytes;
  if (span > kWinBytes) span = kWinBytes;
  if (lo + span > len) span = len - lo;
  src.lo = lo; src.span = span;
  const bool aligned = ((reinterpret_cast<uintptr_t>(buf) + lo) & 15u) == 0;
  const uint32_t nvec = aligned ? uint32_t(span >> 4) : 0u;
  const uint4 *g = reinterpret_cast<const uint4 *>(buf + lo);
  uint4 *w = reinterpret_cast<uint4 *>(win);
  for (uint32_t v = threadIdx.x; v < nvec; v += kTokThreads) w[v] = __ldg(g + v);
  for (uint32_t k = (nvec << 4) + threadIdx.x; k < uint32_t(span); k += kTokThreads) win[k] = __ldg(buf + lo + k);
  if (*fast && threadIdx.x < kWinMargin) win[uint32_t(span) + threadIdx.x] = 0x20;  // (only the end of the document is ever looked at there)
  __syncthreads();
  return src;
}

// ---- A
__global__ void __launch_bounds__(kTokThreads) token_scan_kernel(const uint8_t *buf, uint64_t len, const uint32_t *idx, uint32_t n, uint8_t *type,
                                                                unsigned long long *payload, unsigned long long *tile_bytes, uint32_t *tile_strings,
                                                                TokenTotals *tot, int stage) {
  __shared__ __align__(16) uint8_t win[kWinBytes];  // (stage_window: span + margin <= kWinBytes when it pads)
  __shared__ unsigned long long sh[kTokThreads / 32];
  const uint32_t i0 = blockIdx.x * uint32_t(kTokThreads), i = i0 + threadIdx.x;
  unsigned long long bytes = 0, nstr = 0;
  tok::WindowSrc src;
  bool fast = false;
  if (stage) {
    src = stage_window(buf, len, idx, n, i0, win, &fast);
  } else {
    src.buf = buf; src.len = len; src.win = win; src.lo = 0; src.span = 0;
  }
  const unsigned lane = threadIdx.x & 31u;
  uint32_t t = 0xFFFFFFFFu;  // no token (beyond n)
  unsigned long long v = 0;
  const uint64_t p = i < n ? uint64_t(idx[i]) : 0;
  if (i < n) {
    if (fast) {  // (uniform) the usual case: 32-bit offsets into the window, nothing to check
      const tok::FastWin f{win, uint32_t(src.span)};
      t = tok::classify_token(f, f.limit, uint32_t(p - src.lo), &v, uint32_t(kLaneBudget));
      if (t == 'd') v += src.lo;  // (a float's payload is a document offset)
    } else {
      t = tok::classify_token(src, len, p, &v, kLaneBudget);
    }
  }
  // long strings: one after the other by the whole warp
  uint32_t pending = __ballot_sync(0xFFFFFFFFu, t == tok::kLongString);
  while (pending) {
    const int l = __ffs(int(pending)) - 1;
    pending &= pending - 1;
    const uint64_t pl = __shfl_sync(0xFFFFFFFFu, (unsigned long long)p, l);
    const long long ul = tok::warp_string<false>(src, len, pl, nullptr, lane);
    if (int(lane) == l) {
      if (ul < 0) { t = 0; v = ul == -1 ? uint32_t(tok::kStringError) : uint32_t(tok::kUnclosedStringError); }
      else { t = '"'; v = (unsigned long long)ul | kLongFlag; }
    }
  }
  if (i < n) {
    if (t == '"') {
      bytes = (v & ~kLongFlag) + 5;
      nstr = 1;
    }
    type[i] = uint8_t(t);
    payload[i] = v;
    if (t == 0) atomicMin(&tot->first_error, ((unsigned long long)i << 8) | (v & 0xFFull));
  }
  const unsigned long long tb = block_sum_u64(bytes, sh);
  const unsigned long long ts = block_sum_u64(nstr, sh);
  if (threadIdx.x == 0) {
    tile_bytes[blockIdx.x] = tb;
    tile_strings[blockIdx.x] = uint32_t(ts);
  }
}

// ---- S: exclusive scan of tile_bytes in place (one CTA), totals.  In a sharded pass it also publishes the shard's record
// and summary (sjb200_params.h) into every rank's window: everything they carry is known here -- A's atomicMin have all
// landed (A ran before S on the stream), the totals are this kernel's.  It stores and leaves; nothing waits for a peer.
__global__ void __launch_bounds__(1024) tile_scan_kernel(unsigned long long *tile_bytes, const uint32_t *tile_strings, uint32_t ntiles, TokenTotals *tot,
                                                         TokXchg x) {
  __shared__ unsigned long long sh[32];
  __shared__ unsigned long long carry;
  __shared__ uint32_t shs[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  uint32_t nstr = 0;
  for (uint32_t b = 0; b < ntiles; b += 1024) {
    const uint32_t i = b + threadIdx.x;
    const unsigned long long v = i < ntiles ? tile_bytes[i] : 0ull;
    if (i < ntiles) nstr += tile_strings[i];
    unsigned long long x = v;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
      if (int(threadIdx.x & 31) >= d) x += y;
    }
    if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      unsigned long long w = sh[threadIdx.x];
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, w, d);
        if (int(threadIdx.x) >= d) w += y;
      }
      sh[threadIdx.x] = w;
    }
    __syncthreads();
    const unsigned long long before = carry + ((threadIdx.x >> 5) ? sh[(threadIdx.x >> 5) - 1] : 0ull) + (x - v);
    if (i < ntiles) tile_bytes[i] = before;
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[31];
    __syncthreads();
  }
  for (int d = 16; d > 0; d >>= 1) nstr += __shfl_down_sync(0xFFFFFFFFu, nstr, d);
  if ((threadIdx.x & 31) == 0) shs[threadIdx.x >> 5] = nstr;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
    for (int w = 0; w < 32; w++) s += shs[w];
    tot->n_strings = s;
    tot->string_bytes = carry;
    if (x.xchg.nranks != 0) {
      const unsigned long long fe = tot->first_error;
      const uint32_t w[kSumWords] = {uint32_t(x.len), x.n, s, fe == ~0ull ? 0xFFFFFFFFu : uint32_t(fe >> 8), fe == ~0ull ? 0u : uint32_t(fe & 0xFFull),
                                     uint32_t(carry), uint32_t(carry >> 32), 0u};
      const unsigned long long w0 = xchg_word0(x.xchg.seq, carry),
                               w1 = xchg_word1(x.xchg.seq, x.state_in, 0, carry > x.capacity ? kTokShortFlag : 0u, kTokens);
#pragma unroll
      for (uint32_t r = 0; r < uint32_t(kMaxRanks); r++) {  // (unrolled: x.xchg.peer stays in the parameter space, no stack copy)
        if (r >= x.xchg.nranks) break;
        unsigned long long *sum = x.xchg.peer[r] + xchg_summary_at(x.xchg.seq, x.xchg.rank);
        for (int k = 0; k < kSumWords; k++) {
          const unsigned long long v = (static_cast<unsigned long long>(x.xchg.seq) << 32) | w[k];
          asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(sum + k), "l"(v) : "memory");
        }
        unsigned long long *rec = x.xchg.peer[r] + (size_t(x.xchg.slot) * kMaxRanks + x.xchg.rank) * 2;
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(rec), "l"(w0) : "memory");
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(rec + 1), "l"(w1) : "memory");
      }
    }
  }
}

// ---- B
__global__ void __launch_bounds__(kTokThreads) string_write_kernel(const uint8_t *buf, uint64_t len, const uint32_t *idx, uint32_t n, const uint8_t *type,
                                                                  unsigned long long *payload, const unsigned long long *tile_off, uint32_t ntiles,
                                                                  uint8_t *strbuf, unsigned long long capacity, const TokenTotals *tot, int stage) {
  __shared__ __align__(16) uint8_t win[kWinBytes];  // (stage_window: span + margin <= kWinBytes when it pads)
  __shared__ __align__(16) uint8_t outb[kOutBytes + 16];
  __shared__ unsigned long long sh[kTokThreads / 32];
  const unsigned long long total = tot->string_bytes;
  const uint32_t i0 = blockIdx.x * uint32_t(kTokThreads), i = i0 + threadIdx.x;
  if (total > capacity) {  // CAPACITY: nothing is written, payloads keep the lengths (without the marker of the long ones)
    if (i < n && type[i] == '"') payload[i] &= ~kLongFlag;
    return;
  }
  const unsigned long long t_off = tile_off[blockIdx.x];
  const unsigned long long t_bytes = (blockIdx.x + 1 < ntiles ? tile_off[blockIdx.x + 1] : total) - t_off;  // this tile's records
  if (t_bytes == 0) return;  // (uniform) no string in this tile
  tok::WindowSrc src;
  bool fast = false;
  if (stage) {
    src = stage_window(buf, len, idx, n, i0, win, &fast);
  } else {
    src.buf = buf; src.len = len; src.win = win; src.lo = 0; src.span = 0;
  }
  const unsigned lane = threadIdx.x & 31u;
  const bool mine_is_string = i < n && type[i] == '"';
  const unsigned long long pl0 = mine_is_string ? payload[i] : 0ull;
  const bool mine_is_long = (pl0 & kLongFlag) != 0;
  const unsigned long long ul = pl0 & ~kLongFlag;
  const unsigned long long mine = mine_is_string ? ul + 5 : 0ull;
  // exclusive prefix over the CTA's threads (thread order = document order)
  unsigned long long x = mine;
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
    if (int(threadIdx.x & 31) >= d) x += y;
  }
  if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = x;
  __syncthreads();
  unsigned long long rel = x - mine;  // bytes of this tile's records before mine
  for (uint32_t w = 0; w < (threadIdx.x >> 5); w++) rel += sh[w];
  // the tile's records are composed in shared memory at the destination's phase modulo 16, so that the aligned 16-byte
  // groups of the two coincide, and leave as vectors; a tile with more record bytes than fit writes them directly
  uint8_t *dst_tile = strbuf + t_off;
  const uint32_t phase = uint32_t(reinterpret_cast<uintptr_t>(dst_tile) & 15u);
  const bool staged_out = stage && t_bytes <= kOutBytes;
  uint8_t *rec = staged_out ? outb + phase + rel : dst_tile + rel;
  const uint64_t p = mine_is_string ? uint64_t(idx[i]) : 0;
  if (mine_is_string) {
    rec[0] = uint8_t(ul); rec[1] = uint8_t(ul >> 8); rec[2] = uint8_t(ul >> 16); rec[3] = uint8_t(ul >> 24);
    if (!mine_is_long) {
      if (fast) {
        const tok::FastWin f{win, uint32_t(src.span)};
        tok::walk_string<true>(f, f.limit, uint32_t(p - src.lo), rec + 4);
      } else {
        tok::walk_string<true>(src, len, p, rec + 4);
      }
    }
    rec[4 + ul] = 0;
    payload[i] = t_off + rel;
  }
  uint32_t pending = __ballot_sync(0xFFFFFFFFu, mine_is_long);
  while (pending) {  // long strings: copied by the whole warp
    const int l = __ffs(int(pending)) - 1;
    pending &= pending - 1;
    const uint64_t pl = __shfl_sync(0xFFFFFFFFu, (unsigned long long)p, l);
    uint8_t *dl = reinterpret_cast<uint8_t *>(__shfl_sync(0xFFFFFFFFu, (unsigned long long)reinterpret_cast<uintptr_t>(rec + 4), l));
    tok::warp_string<true>(src, len, pl, dl, lane);
  }
  if (!staged_out) return;
  __syncthreads();
  const uint32_t nb = uint32_t(t_bytes);
  const uint32_t head = (nb < ((16u - phase) & 15u)) ? nb : ((16u - phase) & 15u);  // bytes before the first aligned group
  const uint32_t nvec = (nb - head) >> 4;
  const uint32_t tail = nb - head - (nvec << 4);
  if (threadIdx.x < head) dst_tile[threadIdx.x] = outb[phase + threadIdx.x];
  const uint4 *sv = reinterpret_cast<const uint4 *>(outb + phase + head);  // (phase + head) % 16 == 0
  uint4 *gv = reinterpret_cast<uint4 *>(dst_tile + head);
  for (uint32_t v = threadIdx.x; v < nvec; v += kTokThreads) gv[v] = sv[v];
  if (threadIdx.x < tail) dst_tile[head + (nvec << 4) + threadIdx.x] = outb[phase + head + (nvec << 4) + threadIdx.x];
}

}  // namespace

size_t tokens_scratch_bytes(uint32_t n) {
  const size_t tiles = (size_t(n) + kTokThreads - 1) / kTokThreads;
  return tiles * (sizeof(unsigned long long) + sizeof(uint32_t)) + 64;
}

cudaError_t launch_tile_scan(unsigned long long *tile_sums, const uint32_t *tile_counts, uint32_t ntiles, TokenTotals *tot, cudaStream_t stream) {
  tile_scan_kernel<<<1, 1024, 0, stream>>>(tile_sums, tile_counts, ntiles, tot, TokXchg{});
  return cudaGetLastError();
}

cudaError_t launch_tokens(const uint8_t *buf, uint64_t len, const uint32_t *idx, uint32_t n, uint8_t *type, uint64_t *payload, uint8_t *strbuf,
                          uint64_t strbuf_capacity, void *scratch, TokenTotals *tot_dev, int stage, cudaStream_t stream, const TokXchg *xchg) {
  const uint32_t tiles = uint32_t((size_t(n) + kTokThreads - 1) / kTokThreads);
  unsigned long long *tile_bytes = static_cast<unsigned long long *>(scratch);
  uint32_t *tile_strings = reinterpret_cast<uint32_t *>(tile_bytes + tiles);
  TokXchg x{};
  if (xchg) x = *xchg;
  cudaError_t e = cudaMemsetAsync(tot_dev, 0xFF, sizeof(TokenTotals), stream);  // first_error = ~0; the scan kernel stores the other fields
  if (e != cudaSuccess) return e;
  if (n == 0) {
    tile_scan_kernel<<<1, 1024, 0, stream>>>(tile_bytes, tile_strings, 0, tot_dev, x);
    return cudaGetLastError();
  }
  token_scan_kernel<<<tiles, kTokThreads, 0, stream>>>(buf, len, idx, n, type, reinterpret_cast<unsigned long long *>(payload), tile_bytes, tile_strings, tot_dev,
                                                       stage);
  tile_scan_kernel<<<1, 1024, 0, stream>>>(tile_bytes, tile_strings, tiles, tot_dev, x);
  string_write_kernel<<<tiles, kTokThreads, 0, stream>>>(buf, len, idx, n, type, reinterpret_cast<unsigned long long *>(payload), tile_bytes, tiles, strbuf,
                                                         strbuf_capacity, tot_dev, stage);
  return cudaGetLastError();
}

}  // namespace sjb200
