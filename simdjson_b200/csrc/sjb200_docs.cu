// sjb200_docs.cu -- what follows the scan for streams of documents, on the device (SURVEY.md section 8(f) rows 1 and 3):
//
//   * stream_finish_kernel: the streaming branches of json_structural_indexer::finish
//     (src/generic/stage1/json_structural_indexer.h L249-343) with find_next_document_index
//     (src/generic/stage1/find_next_document_index.h L39-98) on the device-resident index array: one small launch queued
//     right behind the scan -- no host round trip between the scan and its epilogue, no tail gathered to the host.
//   * document table: every place where a document of a whitespace-separated stream starts, as
//     (structural index, byte offset) pairs in stream order -- what lets a consumer fan the documents of one big
//     stage-1 pass out over cores instead of discovering them window by window the way document_stream does
//     (include/simdjson/dom/document_stream-inl.h L245-271).
//   * RS (RFC 7464) and comma-delimited filters: find_next_document_index_json_sequence (L126-267) and
//     filter_comma_delimited (L288-369) as device compactions of the index array, so that those modes no longer copy
//     the document and the index array to the host and back.
//
// A structural's "role" is a function of the byte it points at; a document starts at structural i >= 1 when i is a
// value or an opening bracket and structural i-1 is neither an opening bracket nor a ',' / ':' (the predicate the
// reference's backward walk applies, find_next_document_index.h L60-88).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "sjb200_common.h"
#include "sjb200_docs.h"
#include "sjb200_params.h"

namespace sjb200 {

namespace {

enum : uint32_t { kRoleValue = 0, kRoleSep, kRoleOpenObj, kRoleCloseObj, kRoleOpenArr, kRoleCloseArr };

__device__ __forceinline__ uint32_t role_of(uint32_t c) {
  switch (c) {
    case ':': case ',': return kRoleSep;
    case '{': return kRoleOpenObj;
    case '}': return kRoleCloseObj;
    case '[': return kRoleOpenArr;
    case ']': return kRoleCloseArr;
    default: return kRoleValue;
  }
}
__device__ __forceinline__ bool starts_document(uint32_t cur, uint32_t before) {
  if (cur == kRoleSep || cur == kRoleCloseObj || cur == kRoleCloseArr) return false;
  return !(before == kRoleOpenObj || before == kRoleOpenArr || before == kRoleSep);
}
__device__ __forceinline__ int net_obj(uint32_t r) { return r == kRoleOpenObj ? 1 : (r == kRoleCloseObj ? -1 : 0); }
__device__ __forceinline__ int net_arr(uint32_t r) { return r == kRoleOpenArr ? 1 : (r == kRoleCloseArr ? -1 : 0); }

constexpr int kFinishThreads = 1024;

// block-wide reductions of one CTA of kFinishThreads threads
__device__ int block_sum(int v, int *sh) {
  for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, d);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = 0;
  for (int w = 0; w < kFinishThreads / 32; w++) s += sh[w];
  return s;
}
__device__ int block_max(int v, int *sh) {
  for (int d = 16; d > 0; d >>= 1) v = max(v, __shfl_down_sync(0xFFFFFFFFu, v, d));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = -1;
  for (int w = 0; w < kFinishThreads / 32; w++) s = max(s, sh[w]);
  return s;
}

// The backward walk of find_next_document_index (find_next_document_index.h L39-98) on a device-resident array: from
// structural n-1 back in windows of kFinishThreads structurals until a window holds a document start i >= 1; one CTA.
// Every thread gets *start = that i (-1 when there is none) and the object / array bracket nets of structurals
// [*start, n), or of [0, n) when there is no start.
__device__ void last_document_start(const uint8_t *buf, const uint32_t *idx, uint32_t n, int *sh, int *start, int *nobj_out, int *narr_out) {
  int nobj = 0, narr = 0;  // opens minus closes over the structurals after the current window
  uint32_t hi = n;
  *start = -1;
  for (;;) {
    if (hi == 0) break;
    const uint32_t lo = hi > uint32_t(kFinishThreads) ? hi - uint32_t(kFinishThreads) : 0u;
    const uint32_t i = lo + threadIdx.x;
    const bool in = i < hi;
    uint32_t r = kRoleValue, before = kRoleSep;
    if (in) {
      r = role_of(buf[idx[i]]);
      if (i > 0) before = role_of(buf[idx[i - 1]]);
    }
    const bool is_start = in && i >= 1 && starts_document(r, before);
    const int last = block_max(is_start ? int(i) : -1, sh);
    if (last >= 0) {  // the last document starts at `last`
      const bool tail = in && int(i) >= last;
      nobj += block_sum(tail ? net_obj(r) : 0, sh);
      narr += block_sum(tail ? net_arr(r) : 0, sh);
      *start = last;
      break;
    }
    nobj += block_sum(in ? net_obj(r) : 0, sh);
    narr += block_sum(in ? net_arr(r) : 0, sh);
    hi = lo;
  }
  *nobj_out = nobj;
  *narr_out = narr;
}

// complete_document_count: the number of structurals that belong to complete documents (to every thread).  The last
// document is complete iff its brackets balance; without an internal start it is one document from structural 0 on.
__device__ uint32_t complete_count(const uint8_t *buf, const uint32_t *idx, uint32_t n, int *sh) {
  if (n == 0) return 0;
  int start, nobj, narr;
  last_document_start(buf, idx, n, sh, &start, &nobj, &narr);
  return (nobj == 0 && narr == 0) ? n : (start >= 0 ? uint32_t(start) : 0u);
}

// the streaming branches of finish() (modes 1 and 2) behind a device-resident scan
__global__ void __launch_bounds__(kFinishThreads) stream_finish_kernel(const uint8_t *buf, uint32_t *idx, const Carry *carry, uint32_t len, int mode,
                                                                      StreamFinish *out_dev, StreamFinish *out_host) {
  __shared__ int sh[kFinishThreads / 32];
  const uint64_t count = carry->count;
  const uint32_t state = carry->state, flags = carry->flags;
  StreamFinish res;
  res.err = kSuccess; res.n = 0; res.n_written = 0; res.reserved = 0;
  const bool unclosed = (state >> 1) & 1u;
  bool done = false;
  if (flags & kFlagInternal) { res.err = kUnexpectedError; done = true; }
  else if (flags & kFlagCtl) { res.err = kUnescapedChars; done = true; }  // L261-263: n is left untouched
  uint32_t n = uint32_t(count);
  if (!done) {
    res.n = n; res.n_written = 1;  // sentinels were stored by the scan (L284-286)
    if (n == 0) { res.err = kEmpty; done = true; }  // L289-291
  }
  if (!done) {
    if (mode == kStreamingPartial) {  // L295-317
      if (unclosed) { n--; res.n = n; if (n == 0) { res.err = kCapacity; done = true; } }
      if (!done) {
        const uint32_t m = complete_count(buf, idx, n, sh);
        if (m == 0 && n > 0) {
          if (idx[0] == 0) { res.err = kCapacity; }
          else { res.n = 0; res.err = kEmpty; }
          done = true;
        } else {
          res.n = m;
        }
      }
    } else {  // kStreamingFinal, L318-343
      if (unclosed) n--;
      const uint32_t m = complete_count(buf, idx, n, sh);
      res.n = m;
      __syncthreads();
      if (threadIdx.x == 0) { idx[m + 1] = idx[m]; idx[m] = len; }
      if (m == 0) { res.err = kEmpty; done = true; }
    }
  }
  if (!done && (flags & kFlagUtf8)) res.err = kUtf8Error;  // L395-396
  if (threadIdx.x == 0) {
    *out_dev = res;
    if (out_host) *out_host = res;
  }
}

// The summary of one shard for the extra round of a sharded streaming pass: walk back from the shard's last kept
// structural to its last internal document start (index >= 1), then store the kSumWords-word summary (sjb200_params.h)
// into every rank's window at word `at` (this rank's block).  kept = the shard's structurals, less the stream's last one
// when the stream ends inside a string and this shard holds it; walk = 0 (regular mode) skips the walk.
__global__ void __launch_bounds__(kFinishThreads) stream_summary_kernel(const uint8_t *buf, const uint32_t *idx, uint32_t count, uint32_t kept, uint32_t len,
                                                                       int walk, const __grid_constant__ Xchg x, size_t at) {
  __shared__ int sh[kFinishThreads / 32];
  int start = -1, nobj = 0, narr = 0;
  if (walk && kept > 0) last_document_start(buf, idx, kept, sh, &start, &nobj, &narr);
  const uint32_t r = threadIdx.x;
  if (r < x.nranks) {
    uint32_t w[kSumWords];
    w[0] = len;
    w[1] = count ? idx[0] : 0u;
    w[2] = count ? idx[count - 1] : 0u;
    w[3] = start >= 0 ? uint32_t(start) : 0u;
    w[4] = start >= 0 ? idx[start] : 0u;
    w[5] = uint32_t(nobj);
    w[6] = uint32_t(narr);
    w[7] = (kept ? role_of(buf[idx[0]]) | (role_of(buf[idx[kept - 1]]) << 3) : 0u) | (start >= 0 ? 1u << 6 : 0u);
    unsigned long long *rec = x.peer[r] + at;
    for (int k = 0; k < kSumWords; k++) {
      const unsigned long long v = (static_cast<unsigned long long>(x.seq) << 32) | w[k];
      asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(rec + k), "l"(v) : "memory");
    }
  }
}

// a sharded streaming pass's rewrite of the words it holds (at most two)
__global__ void store_words_kernel(uint32_t *idx, uint32_t nw, uint32_t p0, uint32_t v0, uint32_t p1, uint32_t v1) {
  if (nw > 0) idx[p0] = v0;
  if (nw > 1) idx[p1] = v1;
}

// ---------------------------------------------------------------------------------------------- document table
constexpr int kTabThreads = 256, kTabPerThread = 8, kTabTile = kTabThreads * kTabPerThread;

// first_starts: whether structural 0 starts a document (always, for a whole stream; for a shard, by the predicate
// applied across the cut)
__device__ __forceinline__ bool doc_start_at(const uint8_t *buf, const uint32_t *idx, uint32_t i, bool first_starts) {
  if (i == 0) return first_starts;
  return starts_document(role_of(buf[idx[i]]), role_of(buf[idx[i - 1]]));
}
__global__ void __launch_bounds__(kTabThreads) doc_count_kernel(const uint8_t *buf, const uint32_t *idx, uint32_t n, bool first_starts, uint32_t *tile_count) {
  __shared__ uint32_t sh[kTabThreads / 32];
  const uint32_t base = blockIdx.x * kTabTile;
  uint32_t c = 0;
  for (int k = 0; k < kTabPerThread; k++) {
    const uint32_t i = base + k * kTabThreads + threadIdx.x;
    if (i < n && doc_start_at(buf, idx, i, first_starts)) c++;
  }
  for (int d = 16; d > 0; d >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, d);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
    for (int w = 0; w < kTabThreads / 32; w++) s += sh[w];
    tile_count[blockIdx.x] = s;
  }
}
// exclusive scan of the tile counts in place, one CTA; total -> *ndocs
__global__ void __launch_bounds__(1024) doc_scan_kernel(uint32_t *tile_count, uint32_t ntiles, uint32_t *ndocs) {
  __shared__ uint32_t sh[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t b = 0; b < ntiles; b += 1024) {
    const uint32_t i = b + threadIdx.x;
    const uint32_t v = i < ntiles ? tile_count[i] : 0u;
    uint32_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
      if (int(threadIdx.x & 31) >= d) x += y;
    }
    if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t w = sh[threadIdx.x];
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, d);
        if (int(threadIdx.x) >= d) w += y;
      }
      sh[threadIdx.x] = w;
    }
    __syncthreads();
    const uint32_t before = carry + ((threadIdx.x >> 5) ? sh[(threadIdx.x >> 5) - 1] : 0u) + (x - v);
    if (i < ntiles) tile_count[i] = before;
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) *ndocs = carry;
}
__global__ void __launch_bounds__(kTabThreads) doc_write_kernel(const uint8_t *buf, const uint32_t *idx, uint32_t n, bool first_starts,
                                                               const uint32_t *tile_offset, sjb200_doc_boundary_t *table, uint32_t capacity) {
  __shared__ uint32_t warp_base[kTabThreads / 32];
  __shared__ uint32_t running;
  if (threadIdx.x == 0) running = tile_offset[blockIdx.x];
  __syncthreads();
  const uint32_t base = blockIdx.x * kTabTile;
  for (int k = 0; k < kTabPerThread; k++) {  // consecutive threads take consecutive structurals: table order = stream order
    const uint32_t i = base + k * kTabThreads + threadIdx.x;
    const bool f = i < n && doc_start_at(buf, idx, i, first_starts);
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, f);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_base[warp] = __popc(bal);
    __syncthreads();
    uint32_t off = running;
    for (uint32_t w = 0; w < warp; w++) off += warp_base[w];
    if (f) {
      const uint32_t slot = off + __popc(bal & ((1u << lane) - 1u));
      if (slot < capacity) { table[slot].index = i; table[slot].byte = idx[i]; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t s = 0;
      for (int w = 0; w < kTabThreads / 32; w++) s += warp_base[w];
      running += s;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------- RS / comma filters
// find_next_document_index_json_sequence (find_next_document_index.h L126-267) and filter_comma_delimited (L288-369) as
// compactions of the index array: every thread takes kFltPerThread CONSECUTIVE structurals, a tile is kFltTile of them;
// pass A counts what each tile keeps (and, for the comma format, first the bracket depth entering each tile), one CTA
// scans the tile counts, pass B writes the kept indexes into a second array in order.
constexpr int kFltThreads = 256, kFltPerThread = 8, kFltTile = kFltThreads * kFltPerThread;

__device__ __forceinline__ bool is_ws(uint32_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }

// exclusive prefix of v over the CTA's threads (thread order); *total = sum.  sh: kFltThreads / 32 + 1 ints
__device__ int block_excl_scan(int v, int *sh, int *total) {
  int x = v;
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
    if (int(threadIdx.x & 31) >= d) x += y;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = x;
  __syncthreads();
  int before = 0, sum = 0;
  for (int w = 0; w < kFltThreads / 32; w++) {
    if (w < int(threadIdx.x >> 5)) before += sh[w];
    sum += sh[w];
  }
  *total = sum;
  return before + x - v;
}

// ---- comma-delimited: depth entering each tile
__global__ void __launch_bounds__(kFltThreads) comma_depth_kernel(const uint8_t *buf, const uint32_t *idx, uint32_t n, int *tile_depth) {
  __shared__ int sh[kFltThreads / 32 + 1];
  const uint32_t first = blockIdx.x * kFltTile + threadIdx.x * kFltPerThread;
  int d = 0;
  for (int k = 0; k < kFltPerThread; k++) {
    const uint32_t i = first + k;
    if (i < n) { const uint32_t r = role_of(buf[idx[i]]); d += net_obj(r) + net_arr(r); }
  }
  int total;
  block_excl_scan(d, sh, &total);
  if (threadIdx.x == 0) tile_depth[blockIdx.x] = total;
}
// exclusive scan of ints in place (one CTA); *total_out = sum (may be null)
__global__ void __launch_bounds__(1024) int_scan_kernel(int *v, uint32_t count, int *total_out) {
  __shared__ int sh[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t b = 0; b < count; b += 1024) {
    const uint32_t i = b + threadIdx.x;
    const int val = i < count ? v[i] : 0;
    int x = val;
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
      if (int(threadIdx.x & 31) >= d) x += y;
    }
    if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = sh[threadIdx.x];
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, w, d);
        if (int(threadIdx.x) >= d) w += y;
      }
      sh[threadIdx.x] = w;
    }
    __syncthreads();
    const int before = carry + ((threadIdx.x >> 5) ? sh[(threadIdx.x >> 5) - 1] : 0) + (x - val);
    if (i < count) v[i] = before;
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[31];
    __syncthreads();
  }
  if (threadIdx.x == 0 && total_out) *total_out = carry;
}

// What structural i contributes to the filtered array: 0 or 1 entries (value in *out).  RS format: RS entries go; the
// leader of a run "RS (ws | RS)*" counts the run's separators and, when a scalar is glued to the run's end (stage 1 sees
// RS as a scalar byte, so that value has no index of its own), contributes the value's position.  lead_end (a shard of a
// sharded pass entered inside a separator run of an earlier shard, else 0): the end of the shard's leading whitespace /
// RS run, found by the lead step of filter_pass_kernel, which also counts that run; the RS entries before it are
// absorbed.  A shard's walk stops at its end (len); the shard where the run ends adds the scalar glued to it.
__device__ __forceinline__ bool ws_or_rs(uint32_t c) { return is_ws(c) || c == 0x1E; }
__device__ __forceinline__ int rs_entry(const uint8_t *buf, uint32_t len, const uint32_t *idx, uint32_t n, uint32_t i, uint32_t lead_end, uint32_t *out,
                                        uint32_t *seps, uint32_t *last_sep) {
  const uint32_t at = idx[i];
  if (buf[at] != 0x1E) { *out = at; return 1; }
  if (i == 0 && at < lead_end) return 0;  // (a later RS of the leading run follows an absorbed one: the check below)
  if (i > 0 && buf[idx[i - 1]] == 0x1E) {  // inside the run an earlier RS entry leads?
    bool same = true;
    for (uint32_t q = idx[i - 1] + 1; q < at && same; q++) same = is_ws(buf[q]) || buf[q] == 0x1E;
    if (same) return 0;
  }
  uint32_t s = 1, last = at, v = at + 1;
  while (v < len && ws_or_rs(buf[v])) {
    if (buf[v] == 0x1E) { s++; last = v; }
    v++;
  }
  *seps += s;
  *last_sep = max(*last_sep, last);
  if (v < len && role_of(buf[v]) == kRoleValue) {
    uint32_t j = i + 1;
    while (j < n && idx[j] < v) j++;
    if (!(j < n && idx[j] == v)) { *out = v; return 1; }
  }
  return 0;
}
// the lead step of a shard entered inside a run (run_in): the separators of its leading run and the scalar glued to the
// run's end, unless the shard's scan emitted that byte; *lead_end = the run's end.  One thread walks the run, like the
// leader walk of a run inside a shard.
__device__ __forceinline__ int rs_lead(const uint8_t *buf, uint32_t len, const uint32_t *idx, uint32_t n, uint32_t *out, uint32_t *seps, uint32_t *last_sep,
                                       uint32_t *lead_end) {
  uint32_t v = 0;
  for (; v < len && ws_or_rs(buf[v]); v++)
    if (buf[v] == 0x1E) { (*seps)++; *last_sep = max(*last_sep, v); }
  *lead_end = v;
  if (v < len && role_of(buf[v]) == kRoleValue) {
    uint32_t j = 0;
    while (j < n && idx[j] < v) j++;
    if (!(j < n && idx[j] == v)) { *out = v; return 1; }
  }
  return 0;
}

struct FilterTotals {
  uint32_t kept, seps, last_sep, reserved;
};

// pass A (count) and pass B (write) share the per-thread walk; kComma selects the format.  depth_in / run_in: what a
// shard of a sharded pass carries in from the shards before it (0 for a whole stream)
template <bool kComma, bool kWrite>
__global__ void __launch_bounds__(kFltThreads) filter_pass_kernel(const uint8_t *buf, uint32_t len, const uint32_t *idx, uint32_t n, const int *tile_depth,
                                                                 int *tile_count /* A: out; B: exclusive offsets */, uint32_t *dst, FilterTotals *totals,
                                                                 int depth_in, int run_in) {
  __shared__ int sh[kFltThreads / 32 + 1];
  const uint32_t first = blockIdx.x * kFltTile + threadIdx.x * kFltPerThread;
  int depth = 0;
  if (kComma) {
    int d = 0;
    for (int k = 0; k < kFltPerThread; k++) {
      const uint32_t i = first + k;
      if (i < n) { const uint32_t r = role_of(buf[idx[i]]); d += net_obj(r) + net_arr(r); }
    }
    int total;
    depth = depth_in + tile_depth[blockIdx.x] + block_excl_scan(d, sh, &total);
  }
  uint32_t vals[kComma ? kFltPerThread : kFltPerThread + 1];  // (RS: one more for the lead step)
  int cnt = 0;
  uint32_t seps = 0, last_sep = 0;
  uint32_t lead_end = 0;  // (the thread of structural 0 does the lead step; no other thread reads lead_end)
  if (!kComma && run_in && first == 0 && rs_lead(buf, len, idx, n, &vals[0], &seps, &last_sep, &lead_end)) cnt = 1;
  for (int k = 0; k < kFltPerThread; k++) {
    const uint32_t i = first + k;
    if (i >= n) break;
    if (kComma) {
      const uint32_t at = idx[i], c = buf[at], r = role_of(c);
      if (r == kRoleOpenObj || r == kRoleOpenArr) depth++;
      else if (r == kRoleCloseObj || r == kRoleCloseArr) depth--;
      else if (c == ',' && depth == 0) { seps++; last_sep = max(last_sep, at); continue; }
      vals[cnt++] = at;
    } else {
      uint32_t v = 0;
      if (rs_entry(buf, len, idx, n, i, lead_end, &v, &seps, &last_sep)) vals[cnt++] = v;
    }
  }
  int total;
  const int before = block_excl_scan(cnt, sh, &total);
  if (!kWrite) {
    if (threadIdx.x == 0) tile_count[blockIdx.x] = total;
    if (seps) { atomicAdd(&totals->seps, seps); atomicMax(&totals->last_sep, last_sep); }
  } else {
    const uint32_t base = uint32_t(tile_count[blockIdx.x] + before);
    for (int k = 0; k < cnt; k++) dst[base + k] = vals[k];
  }
}

__global__ void copy_kept_kernel(uint32_t *idx, const uint32_t *src, const int *kept_total) {
  const uint32_t kept = uint32_t(*kept_total);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < kept; i += gridDim.x * blockDim.x) idx[i] = src[i];
}

// the tail of finish() for modes 3..6 on the filtered array (json_structural_indexer.h L344-393); `idx` already holds it
__global__ void __launch_bounds__(kFinishThreads) filter_finish_kernel(const uint8_t *buf, uint32_t *idx, const FilterTotals *tot, const int *kept_total, uint32_t len,
                                                                      int mode, uint32_t flags, StreamFinish *out_dev, StreamFinish *out_host) {
  __shared__ int sh[kFinishThreads / 32];
  const uint32_t n = uint32_t(*kept_total), seps = tot->seps, last_sep = tot->last_sep;
  const bool rs = (mode == kJsonSequencePartial || mode == kJsonSequenceFinal);
  const bool is_final = (mode == kJsonSequenceFinal || mode == kCommaDelimitedFinal);
  StreamFinish res;
  res.err = kSuccess; res.n = n; res.n_written = 1; res.reserved = 0;
  uint32_t m = 0, next_start = len;
  bool too_large = false;
  if (n != 0) {
    if (rs) {
      if (seps == 0) m = is_final ? complete_count(buf, idx, n, sh) : 0u;
      else if (is_final) m = n;
      else {
        next_start = last_sep;
        if (seps < 2) too_large = true;
        else {  // entries before the last separator: the array is sorted, a bisection finds the cut
          uint32_t lo = 0, hi = n;
          while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (idx[mid] < last_sep) lo = mid + 1; else hi = mid; }
          m = lo;
        }
      }
    } else {
      if (is_final) m = complete_count(buf, idx, n, sh);
      else if (seps == 0) too_large = true;
      else {
        next_start = last_sep + 1;
        uint32_t lo = 0, hi = n;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (idx[mid] < last_sep) lo = mid + 1; else hi = mid; }
        if (lo != 0) { res.n = lo; m = complete_count(buf, idx, lo, sh); }
      }
    }
  }
  __syncthreads();
  if (!is_final) {  // L344-359, L367-384
    if (too_large) res.err = kCapacity;
    else if (m == 0) { res.n = 0; res.err = kEmpty; }
    else { res.n = m; if (threadIdx.x == 0) idx[m] = next_start; }
  } else {  // L360-366, L385-393
    res.n = m;
    if (threadIdx.x == 0) { idx[m + 1] = idx[m]; idx[m] = len; }  // (idx[m] is whatever the in-place filter left there, as in the reference)
    if (m == 0) res.err = kEmpty;
  }
  if (res.err == kSuccess && (flags & kFlagUtf8)) res.err = kUtf8Error;
  if (threadIdx.x == 0) {
    *out_dev = res;
    if (out_host) *out_host = res;
  }
}

// ---------------------------------------------------------------------------------------------- sharded RS / comma passes
// the extra rounds of a delimited pass (sjb200_comm.cu): every kernel stores its words, tagged with x.seq, into
// every rank's window at word `at` (this rank's block, sjb200_params.h)
__device__ __forceinline__ void store_tagged(const Xchg &x, uint32_t r, size_t at, const uint32_t *w, int nwords) {
  unsigned long long *rec = x.peer[r] + at;
  for (int k = 0; k < nwords; k++) {
    const unsigned long long v = (static_cast<unsigned long long>(x.seq) << 32) | w[k];
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(rec + k), "l"(v) : "memory");
  }
}

// RS carry round, over the whole grid: *other = 1 when a byte after the shard's last structural (byte 0 without one) is
// neither whitespace nor RS.  Threads leave at the first such byte they meet, the others at their next look at *other,
// so a shard that ends in a long string or scalar costs a few strides, one that ends in a long whitespace run one pass.
constexpr int kWsThreads = 256, kWsBlocks = 528, kWsPoll = 16;
__global__ void __launch_bounds__(kWsThreads) trailing_ws_kernel(const uint8_t *buf, const uint32_t *idx, uint32_t n, uint32_t len, int *other) {
  const uint64_t lo = n ? uint64_t(idx[n - 1]) + 1 : 0u, stride = uint64_t(gridDim.x) * blockDim.x;
  uint32_t k = 0;
  for (uint64_t q = lo + uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; q < len; q += stride) {
    if (!ws_or_rs(buf[q])) { atomicOr(other, 1); return; }
    if (++k % kWsPoll == 0 && *reinterpret_cast<volatile int *>(other)) return;
  }
}

// carry round: the shard's length and what the filters of later shards need from it -- comma: the bracket net over its n
// structurals (*depth_total); RS: whether it ends inside a separator run (its last structural is an RS entry followed
// only by whitespace / RS, *other == 0) and whether it is whitespace / RS only
__global__ void delim_carry_kernel(const uint8_t *buf, const uint32_t *idx, uint32_t n, uint32_t len, int comma, const int *depth_total, const int *other,
                                   const __grid_constant__ Xchg x, size_t at) {
  const bool ok = comma || *other == 0;
  if (threadIdx.x < x.nranks) {
    uint32_t w[kDelimCarryWords];
    w[0] = len;
    w[1] = comma ? uint32_t(*depth_total) : uint32_t(n > 0 && buf[idx[n - 1]] == 0x1E && ok);
    w[2] = comma ? 0u : uint32_t(n == 0 && ok);
    store_tagged(x, threadIdx.x, at, w, kDelimCarryWords);
  }
}

// filter round: {filtered entries, separators, last separator, filtered entries before it} -> out4
__global__ void delim_totals_kernel(const uint32_t *dst, const int *kept_total, const FilterTotals *tot, uint32_t *out4) {
  if (threadIdx.x != 0) return;
  const uint32_t n = uint32_t(*kept_total), seps = tot->seps, last_sep = tot->last_sep;
  uint32_t lo = 0, hi = seps ? n : 0u;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (dst[mid] < last_sep) lo = mid + 1; else hi = mid; }
  out4[0] = n; out4[1] = seps; out4[2] = last_sep; out4[3] = lo;
}

__global__ void publish_kernel(const uint32_t *src, uint32_t nwords, const __grid_constant__ Xchg x, size_t at) {
  if (threadIdx.x < x.nranks) store_tagged(x, threadIdx.x, at, src, int(nwords));
}

// tail round: the (at most three) words n, n+1, n+2 of the whole call this rank holds, read before the filtered entries
// go back into idx -- a word past the filtered array is what the scan left there (a raw structural, as after the
// reference's in-place filter)
__global__ void delim_tail_kernel(const uint32_t *dst, const uint32_t *idx, DelimTail t, const __grid_constant__ Xchg x, size_t at) {
  uint32_t w[3];
  for (int k = 0; k < 3; k++) w[k] = t.src[k] == 1 ? dst[t.pos[k]] + t.add : (t.src[k] == 2 ? idx[t.pos[k]] + t.add : 0u);
  if (threadIdx.x < x.nranks) store_tagged(x, threadIdx.x, at, w, 3);
}

struct FilterScratch {
  uint32_t *dst;
  int *tile_depth, *tile_count;
  FilterTotals *tot;
  int *kept_total, *depth_total, *other;
  uint32_t *out4;
};
// the scratch of launch_stream_filter (n + 8 words, the two tile arrays, the totals), then the delimited rounds' words
FilterScratch filter_layout(uint32_t *scratch, uint32_t n) {
  const uint32_t ntiles = (n + kFltTile - 1) / kFltTile;
  FilterScratch f;
  f.dst = scratch;
  f.tile_depth = reinterpret_cast<int *>(scratch + size_t(n) + 8);
  f.tile_count = f.tile_depth + ntiles + 4;
  f.tot = reinterpret_cast<FilterTotals *>(f.tile_count + ntiles + 4);
  f.kept_total = reinterpret_cast<int *>(f.tot + 1);
  f.depth_total = f.kept_total + 1;
  f.other = f.kept_total + 2;
  f.out4 = reinterpret_cast<uint32_t *>(f.kept_total + 4);
  return f;
}

}  // namespace

size_t filter_scratch_words(uint32_t n) { return size_t(n) + 8 + 2 * (size_t((n + kFltTile - 1) / kFltTile) + 4) + 8; }

// idx[0, n) (device) -> filtered in place; result (error code, n) in out_dev / out_host.  n = structurals the scan found,
// already reduced by one when the input ended inside a string.  scratch: filter_scratch_words(n) words.
cudaError_t launch_stream_filter(const uint8_t *buf, uint32_t len, uint32_t *idx, uint32_t n, int mode, uint32_t flags, uint32_t *scratch, StreamFinish *out_dev,
                                 StreamFinish *out_host, cudaStream_t stream) {
  const uint32_t ntiles = (n + kFltTile - 1) / kFltTile;
  uint32_t *dst = scratch;                                           // n + 8 words
  int *tile_depth = reinterpret_cast<int *>(scratch + size_t(n) + 8);  // ntiles + 4
  int *tile_count = tile_depth + ntiles + 4;                          // ntiles + 4
  FilterTotals *tot = reinterpret_cast<FilterTotals *>(tile_count + ntiles + 4);
  int *kept_total = reinterpret_cast<int *>(tot + 1);
  cudaError_t e = cudaMemsetAsync(tot, 0, sizeof(FilterTotals) + sizeof(int), stream);
  if (e != cudaSuccess) return e;
  const bool comma = (mode == kCommaDelimitedPartial || mode == kCommaDelimitedFinal);
  if (ntiles) {
    if (comma) {
      comma_depth_kernel<<<ntiles, kFltThreads, 0, stream>>>(buf, idx, n, tile_depth);
      int_scan_kernel<<<1, 1024, 0, stream>>>(tile_depth, ntiles, nullptr);
      filter_pass_kernel<true, false><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, tile_depth, tile_count, dst, tot, 0, 0);
      int_scan_kernel<<<1, 1024, 0, stream>>>(tile_count, ntiles, kept_total);
      filter_pass_kernel<true, true><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, tile_depth, tile_count, dst, tot, 0, 0);
    } else {
      filter_pass_kernel<false, false><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, tile_depth, tile_count, dst, tot, 0, 0);
      int_scan_kernel<<<1, 1024, 0, stream>>>(tile_count, ntiles, kept_total);
      filter_pass_kernel<false, true><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, tile_depth, tile_count, dst, tot, 0, 0);
    }
    // only the kept entries go back: the words behind them keep what the scan left there, like the reference's in-place filter
    copy_kept_kernel<<<std::min<uint32_t>(ntiles, 1024u), 256, 0, stream>>>(idx, dst, kept_total);
  }
  filter_finish_kernel<<<1, kFinishThreads, 0, stream>>>(buf, idx, tot, kept_total, len, mode, flags, out_dev, out_host);
  return cudaGetLastError();
}

cudaError_t launch_stream_finish(const uint8_t *buf, uint32_t *idx, const Carry *carry, uint32_t len, int mode, StreamFinish *out_dev, StreamFinish *out_host,
                                 cudaStream_t stream) {
  stream_finish_kernel<<<1, kFinishThreads, 0, stream>>>(buf, idx, carry, len, mode, out_dev, out_host);
  return cudaGetLastError();
}

size_t doc_table_scratch_words(uint32_t n) { return size_t((n + kTabTile - 1) / kTabTile) + 1; }

cudaError_t launch_doc_table(const uint8_t *buf, const uint32_t *idx, uint32_t n, bool first_starts, uint32_t *scratch, sjb200_doc_boundary_t *table,
                             uint32_t capacity, uint32_t *ndocs_dev, cudaStream_t stream) {
  const uint32_t ntiles = (n + kTabTile - 1) / kTabTile;
  if (ntiles == 0) return cudaMemsetAsync(ndocs_dev, 0, sizeof(uint32_t), stream);
  doc_count_kernel<<<ntiles, kTabThreads, 0, stream>>>(buf, idx, n, first_starts, scratch);
  doc_scan_kernel<<<1, 1024, 0, stream>>>(scratch, ntiles, ndocs_dev);
  doc_write_kernel<<<ntiles, kTabThreads, 0, stream>>>(buf, idx, n, first_starts, scratch, table, capacity);
  return cudaGetLastError();
}

cudaError_t launch_stream_summary(const uint8_t *buf, const uint32_t *idx, uint32_t count, uint32_t kept, uint32_t len, int walk, const Xchg &x,
                                  size_t at, cudaStream_t stream) {
  stream_summary_kernel<<<1, kFinishThreads, 0, stream>>>(buf, idx, count, kept, len, walk, x, at);
  return cudaGetLastError();
}

size_t delim_scratch_words(uint32_t n) { return filter_scratch_words(n) + 8; }

cudaError_t launch_delim_carry(const uint8_t *buf, const uint32_t *idx, uint32_t n, uint32_t len, bool comma, uint32_t *scratch, const Xchg &x,
                               size_t at, cudaStream_t stream) {
  const FilterScratch f = filter_layout(scratch, n);
  const uint32_t ntiles = (n + kFltTile - 1) / kFltTile;
  if (comma) {
    cudaError_t e = cudaMemsetAsync(f.tile_depth, 0, sizeof(int), stream);  // (the filter round's one tile when n = 0)
    if (e == cudaSuccess) e = cudaMemsetAsync(f.depth_total, 0, sizeof(int), stream);
    if (e != cudaSuccess) return e;
    if (ntiles) {  // the tile depths stay in the scratch for the filter round
      comma_depth_kernel<<<ntiles, kFltThreads, 0, stream>>>(buf, idx, n, f.tile_depth);
      int_scan_kernel<<<1, 1024, 0, stream>>>(f.tile_depth, ntiles, f.depth_total);
    }
  } else {
    cudaError_t e = cudaMemsetAsync(f.other, 0, sizeof(int), stream);
    if (e != cudaSuccess) return e;
    trailing_ws_kernel<<<kWsBlocks, kWsThreads, 0, stream>>>(buf, idx, n, len, f.other);
  }
  delim_carry_kernel<<<1, 32, 0, stream>>>(buf, idx, n, len, comma, f.depth_total, f.other, x, at);
  return cudaGetLastError();
}

cudaError_t launch_delim_filter(const uint8_t *buf, uint32_t len, const uint32_t *idx, uint32_t n, bool comma, int depth_in, bool run_in, uint32_t *scratch,
                                uint32_t *totals_host, cudaStream_t stream) {
  const FilterScratch f = filter_layout(scratch, n);
  const uint32_t ntiles = std::max<uint32_t>(1u, (n + kFltTile - 1) / kFltTile);  // the lead step runs even without structurals
  cudaError_t e = cudaMemsetAsync(f.tot, 0, sizeof(FilterTotals) + sizeof(int), stream);
  if (e != cudaSuccess) return e;
  if (comma) {
    filter_pass_kernel<true, false><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, f.tile_depth, f.tile_count, f.dst, f.tot, depth_in, 0);
    int_scan_kernel<<<1, 1024, 0, stream>>>(f.tile_count, ntiles, f.kept_total);
    filter_pass_kernel<true, true><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, f.tile_depth, f.tile_count, f.dst, f.tot, depth_in, 0);
  } else {
    filter_pass_kernel<false, false><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, f.tile_depth, f.tile_count, f.dst, f.tot, 0, run_in);
    int_scan_kernel<<<1, 1024, 0, stream>>>(f.tile_count, ntiles, f.kept_total);
    filter_pass_kernel<false, true><<<ntiles, kFltThreads, 0, stream>>>(buf, len, idx, n, f.tile_depth, f.tile_count, f.dst, f.tot, 0, run_in);
  }
  delim_totals_kernel<<<1, 32, 0, stream>>>(f.dst, f.kept_total, f.tot, f.out4);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return cudaMemcpyAsync(totals_host, f.out4, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
}

const uint32_t *delim_filtered(const uint32_t *scratch) { return scratch; }

cudaError_t launch_delim_publish_totals(uint32_t *scratch, uint32_t n, const Xchg &x, size_t at, cudaStream_t stream) {
  publish_kernel<<<1, 32, 0, stream>>>(filter_layout(scratch, n).out4, 4, x, at);
  return cudaGetLastError();
}

cudaError_t launch_delim_tail(uint32_t *scratch, uint32_t n, uint32_t *idx, const DelimTail &t, bool publish, const Xchg &x, size_t at,
                              cudaStream_t stream) {
  const FilterScratch f = filter_layout(scratch, n);
  if (publish) delim_tail_kernel<<<1, 32, 0, stream>>>(f.dst, idx, t, x, at);
  const uint32_t ntiles = std::max<uint32_t>(1u, (n + kFltTile - 1) / kFltTile);
  copy_kept_kernel<<<std::min<uint32_t>(ntiles + 1, 1024u), 256, 0, stream>>>(idx, f.dst, f.kept_total);
  return cudaGetLastError();
}

cudaError_t launch_store_words(uint32_t *idx, uint32_t nw, uint32_t p0, uint32_t v0, uint32_t p1, uint32_t v1, cudaStream_t stream) {
  store_words_kernel<<<1, 1, 0, stream>>>(idx, nw, p0, v0, p1, v1);
  return cudaGetLastError();
}

}  // namespace sjb200
