// sjb200_grammar.cu -- the nesting grammar of stage 2 for every document of a stream (sjb200_document_errors_dev): the
// tile routines of sjb200_grammar.cuh as sm_90a kernels.  Launch order on one stream: the document-start bitmap, the
// tile records (pass A), the fold tree up and down (pass B), the judgement of every structural (pass C), the results.
#include "sjb200_common.h"
#include "sjb200_grammar.h"

namespace sjb200 {
namespace gram {
namespace {

constexpr unsigned kWarps = 4;  // warps per CTA of the tile and fold kernels

struct Scratch {
  unsigned long long *first;  // [D] (index << 8 | code) of each document's first error
  uint32_t *starts;           // document-start bitmap, bit 0 set
  uint32_t *records;          // the levels of the fold tree, 2 + words per record; level 0: one per tile
  uint32_t *identity;         // one empty record
};

// the last document whose start is <= k (kNone: before the first)
__device__ __forceinline__ uint32_t doc_of(const GrammarArgs &a, uint32_t k) {
  if (!a.docs) return 0;
  uint32_t lo = 0, hi = a.ndocs;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (a.docs[mid].index <= k) lo = mid + 1; else hi = mid;
  }
  return lo == 0 ? kNone : lo - 1;
}

// the bitmap of document starts, and the check of the table (ascending, every entry below n)
__global__ void __launch_bounds__(256) gram_starts_kernel(GrammarArgs a, uint32_t *starts, uint32_t *summary) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) atomicOr(starts, 1u);
  if (!a.docs || i >= a.ndocs) return;
  const uint32_t s = a.docs[i].index;
  if (s >= a.n || (i > 0 && a.docs[i - 1].index >= s)) {
    atomicOr(summary, 1u);
    return;
  }
  atomicOr(starts + (s >> 5), 1u << (s & 31u));
}

__device__ __forceinline__ Grammar grammar_of(const GrammarArgs &a, const Scratch &s, const uint32_t *prefix) {
  Grammar g;
  g.type = a.type;
  g.payload = a.payload;
  g.n = a.n;
  g.starts = s.starts;
  g.whole = a.docs == nullptr;
  g.max_depth = a.max_depth;
  g.words = (a.max_depth + 31) / 32;
  g.prefix = prefix;
  return g;
}

// pass A: one warp per tile
__global__ void __launch_bounds__(kWarps * 32) gram_record_kernel(GrammarArgs a, Scratch s, uint32_t tiles) {
  __shared__ TileSmem<kItems> sm[kWarps];
  const Grammar g = grammar_of(a, s, nullptr);
  const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  for (uint32_t t = blockIdx.x * kWarps + w; t < tiles; t += gridDim.x * kWarps) {
    load_tile<kItems>(g, sm[w], lane, t * kTile);
    tile_record<kItems>(g, sm[w], lane, t * kTile, s.records + size_t(t) * (2 + g.words));
  }
}

struct FoldSmem {
  uint32_t acc[2 + kMaxWords];
  uint32_t child[2 + kMaxWords];
};

// pass B: one warp per group of 32 records
__global__ void __launch_bounds__(kWarps * 32) gram_up_kernel(const uint32_t *level, uint32_t count, uint32_t *up, uint32_t words) {
  __shared__ FoldSmem sm[kWarps];
  const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  const uint32_t groups = (count + 31) / 32;
  for (uint32_t gr = blockIdx.x * kWarps + w; gr < groups; gr += gridDim.x * kWarps)
    fold_up_group(lane, sm[w].acc, sm[w].child, level, count, up, gr, words);
}
__global__ void __launch_bounds__(kWarps * 32) gram_down_kernel(uint32_t *level, uint32_t count, const uint32_t *up, uint32_t words) {
  __shared__ FoldSmem sm[kWarps];
  const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  const uint32_t groups = (count + 31) / 32;
  for (uint32_t gr = blockIdx.x * kWarps + w; gr < groups; gr += gridDim.x * kWarps)
    fold_down_group(lane, sm[w].acc, sm[w].child, level, count, up, gr, words);
}

// pass C: one warp per tile; each document's first error by atomicMin
__global__ void __launch_bounds__(kWarps * 32) gram_check_kernel(GrammarArgs a, Scratch s, uint32_t tiles) {
  __shared__ TileSmem<kItems> sm[kWarps];
  const Grammar g = grammar_of(a, s, s.records);
  const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  auto report = [&](uint32_t pos, uint32_t code, uint32_t index) {
    const uint32_t d = doc_of(a, pos);
    if (d != kNone) atomicMin(s.first + d, (static_cast<unsigned long long>(index) << 8) | code);
  };
  for (uint32_t t = blockIdx.x * kWarps + w; t < tiles; t += gridDim.x * kWarps) {
    load_tile<kItems>(g, sm[w], lane, t * kTile);
    tile_check<kItems>(g, sm[w], lane, t * kTile, t, report);
  }
}

// one result per document, and the two counts
__global__ void __launch_bounds__(256) gram_result_kernel(GrammarArgs a, Scratch s, uint32_t *summary) {
  const uint32_t D = a.docs ? a.ndocs : 1;
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  DocError r;
  if (summary[0]) {
    r = DocError{int32_t(kUnexpected), kNone};
  } else if (a.n == 0) {
    r = DocError{int32_t(kEmpty), 0};
  } else if (s.first[d] != ~0ull) {
    r = DocError{int32_t(s.first[d] & 0xFFu), uint32_t(s.first[d] >> 8)};
  } else {
    r = DocError{0, a.docs && d + 1 < a.ndocs ? a.docs[d + 1].index : a.n};
  }
  a.out[d] = r;
  if (r.error != 0) {
    atomicAdd(summary + 1, 1u);
    atomicMin(summary + 2, d);
  }
}

unsigned grid_for(uint64_t items, uint64_t per_cta, int sm_count, int per_sm) {
  const uint64_t want = (items + per_cta - 1) / per_cta;
  const uint64_t cap = uint64_t(sm_count) * per_sm;
  return unsigned(want < 1 ? 1 : (want < cap ? want : cap));
}

// record counts of the fold tree's levels, from one per tile up to one
int tree_levels(uint32_t tiles, uint32_t *count, int max_levels) {
  int L = 0;
  uint32_t c = tiles;
  for (;;) {
    count[L++] = c;
    if (c <= 1 || L == max_levels) break;
    c = (c + 31) / 32;
  }
  return L;
}

}  // namespace

size_t grammar_scratch_words(uint32_t n, uint32_t ndocs, uint32_t max_depth) {
  const uint32_t D = ndocs ? ndocs : 1;
  const size_t stride = 2 + (max_depth + 31) / 32;
  uint32_t count[8];
  const int L = tree_levels((n + kTile - 1) / kTile, count, 8);
  size_t recs = 1;  // the identity
  for (int l = 0; l < L; l++) recs += count[l];
  return 2 * size_t(D) + (size_t(n) + 31) / 32 + 1 + recs * stride;
}

cudaError_t launch_document_errors(const GrammarArgs &args, uint32_t *scratch, uint32_t *summary, int sm_count, cudaStream_t st, int *launches) {
  const GrammarArgs a = args;
  const uint32_t D = a.docs ? a.ndocs : 1;
  const uint32_t words = (a.max_depth + 31) / 32;
  const size_t stride = 2 + words;
  const uint32_t tiles = (a.n + kTile - 1) / kTile;
  uint32_t count[8];
  const int L = tree_levels(tiles, count, 8);
  Scratch s;
  s.first = reinterpret_cast<unsigned long long *>(scratch);
  s.starts = scratch + 2 * size_t(D);
  const size_t bitmap_words = (size_t(a.n) + 31) / 32 + 1;
  s.records = s.starts + bitmap_words;
  uint32_t *level[8];
  size_t at = 0;
  for (int l = 0; l < L; l++) {
    level[l] = s.records + at * stride;
    at += count[l];
  }
  s.identity = s.records + at * stride;
  const uint32_t init[3] = {0, 0, 0xFFFFFFFFu};
  cudaError_t e = cudaMemsetAsync(scratch, 0xFF, sizeof(unsigned long long) * D, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.starts, 0, sizeof(uint32_t) * bitmap_words, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.identity, 0, sizeof(uint32_t) * stride, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(summary, init, sizeof(init), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  *launches = 2;
  gram_starts_kernel<<<(D + 255) / 256, 256, 0, st>>>(a, s.starts, summary);
  if (tiles) {
    const unsigned tile_grid = grid_for(tiles, kWarps, sm_count, 16);
    gram_record_kernel<<<tile_grid, kWarps * 32, 0, st>>>(a, s, tiles);
    for (int l = 0; l + 1 < L; l++)
      gram_up_kernel<<<grid_for((count[l] + 31) / 32, kWarps, sm_count, 16), kWarps * 32, 0, st>>>(level[l], count[l], level[l + 1], words);
    for (int l = L - 1; l >= 0; l--)
      gram_down_kernel<<<grid_for((count[l] + 31) / 32, kWarps, sm_count, 16), kWarps * 32, 0, st>>>(level[l], count[l],
                                                                                                   l + 1 < L ? level[l + 1] : s.identity, words);
    gram_check_kernel<<<tile_grid, kWarps * 32, 0, st>>>(a, s, tiles);
    *launches += 2 * L + 1;
  }
  gram_result_kernel<<<(D + 255) / 256, 256, 0, st>>>(a, s, summary);
  return cudaGetLastError();
}

// =============================================================================== one rank of a sharded pass
namespace {

struct ShardScratch {
  unsigned long long *first;  // [owned + 1]: each document's first error, then the leading segment's (index << 8 | code)
  uint32_t *tally;            // [0] the table is bad, [1] documents in error but the last, [2] the first of them
  uint32_t *starts;
  uint32_t *records;          // the fold tree's levels, then the incoming record
  uint32_t *incoming;
  uint32_t *level[8];
  uint32_t count[8];
  int L;
};

ShardScratch shard_layout(uint32_t *scratch, uint32_t n, uint32_t ndocs, uint32_t max_depth) {
  ShardScratch s;
  const size_t stride = 2 + (max_depth + 31) / 32;
  const size_t D = (ndocs ? ndocs : 1) + 1;
  s.first = reinterpret_cast<unsigned long long *>(scratch);
  s.tally = scratch + 2 * D;
  s.starts = s.tally + 4;
  s.records = s.starts + (size_t(n) + 31) / 32 + 1;
  s.L = tree_levels((n + kTile - 1) / kTile, s.count, 8);
  size_t at = 0;
  for (int l = 0; l < s.L; l++) {
    s.level[l] = s.records + at * stride;
    at += s.count[l];
  }
  s.incoming = s.records + at * stride;
  return s;
}

__device__ __forceinline__ void store_tagged(const Xchg &x, uint32_t r, size_t at, uint32_t w) {
  sj_st_sys_u64(x.peer[r] + at, (static_cast<unsigned long long>(x.seq) << 32) | w);
}

// the table's check and its start bitmap, as gram_starts_kernel but without bit 0: that one is the stream's
__global__ void __launch_bounds__(256) gram_shard_starts_kernel(GrammarArgs a, uint32_t *starts, uint32_t *tally) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (!a.docs || i >= a.ndocs) return;
  const uint32_t s = a.docs[i].index;
  if (s >= a.n || (i > 0 && a.docs[i - 1].index >= s)) {
    atomicOr(tally, 1u);
    return;
  }
  atomicOr(starts + (s >> 5), 1u << (s & 31u));
}

// edge round and the pass's round-0 record, one thread per rank
__global__ void gram_shard_edges_kernel(GrammarArgs a, int whole, uint32_t max_depth_word, int failed, const uint32_t *tally,
                                        const __grid_constant__ Xchg x, size_t at) {
  const uint32_t r = threadIdx.x;
  if (r >= x.nranks) return;
  const bool table = !failed && !whole && a.docs && a.ndocs;
  uint32_t w[kGramEdgeWords];
  shard_edge_words(a.type, a.n, whole, table ? a.ndocs : 0u, table ? a.docs[0].index : 0u, table ? a.docs[a.ndocs - 1].index : 0u, !failed && *tally,
                   failed, max_depth_word, w);
  for (int k = 0; k < kGramEdgeWords; k++) store_tagged(x, r, at + kGramEdgeAt + k, w[k]);
  unsigned long long *rec = x.peer[r] + (size_t(x.slot) * kMaxRanks + x.rank) * 2;
  sj_st_sys_u64(rec, xchg_word0(x.seq, a.n));
  sj_st_sys_u64(rec + 1, xchg_word1(x.seq, 0, 0, failed ? uint32_t(kFlagInternal) : 0u, kGrammar));
}

__global__ void gram_shard_root_kernel(uint32_t *starts) { atomicOr(starts, 1u); }

__device__ __forceinline__ Grammar shard_grammar(const ShardPass &p, const uint32_t *starts, const uint32_t *prefix) {
  Grammar g;
  g.type = p.a.type;
  g.payload = p.a.payload;
  g.n = p.a.n;
  g.starts = starts;
  g.whole = p.whole;
  g.max_depth = p.a.max_depth;
  g.words = (p.a.max_depth + 31) / 32;
  g.prefix = prefix;
  return g;
}

// pass A with the halo: one warp per tile
__global__ void __launch_bounds__(kWarps * 32) gram_shard_record_kernel(ShardPass p, ShardHalo h, const uint32_t *starts, uint32_t *records, uint32_t tiles) {
  __shared__ TileSmem<kItems> sm[kWarps];
  const Grammar g = shard_grammar(p, starts, nullptr);
  const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  for (uint32_t t = blockIdx.x * kWarps + w; t < tiles; t += gridDim.x * kWarps) {
    load_tile<kItems>(g, sm[w], lane, t * kTile, h);
    tile_record<kItems>(g, sm[w], lane, t * kTile, records + size_t(t) * (2 + g.words), h);
  }
}

// the shard's record (null: the empty record of a shard without structurals) into every window, one warp
__global__ void gram_shard_post_record_kernel(const uint32_t *top, uint32_t words, const __grid_constant__ Xchg x, size_t at) {
  const unsigned lane = threadIdx.x;
  for (uint32_t r = 0; r < x.nranks; r++)
    for (uint32_t k = lane; k < 2 + words; k += 32) store_tagged(x, r, at + kGramRecAt + k, top && (k < 2 || k - 2 < (top[1] + 31) / 32) ? top[k] : 0u);
}

// the stack entering this shard: the records of ranks 0 .. rank - 1 folded in order (the window's words), one warp
__global__ void gram_shard_incoming_kernel(const unsigned long long *win, uint32_t rank, uint32_t words, uint32_t *dst) {
  __shared__ FoldSmem sm;
  shard_incoming(threadIdx.x, sm.acc, sm.child, [&](uint32_t r, uint32_t k) { return uint32_t(win[size_t(r) * kGramWords + kGramRecAt + k]); }, rank, words,
                 dst);
}

// pass C with the halo: the first error of each document that starts here, and of the leading segment (first[owned])
__global__ void __launch_bounds__(kWarps * 32) gram_shard_check_kernel(ShardPass p, ShardHalo h, const uint32_t *starts, const uint32_t *prefix,
                                                                       unsigned long long *first, uint32_t tiles) {
  __shared__ TileSmem<kItems> sm[kWarps];
  const Grammar g = shard_grammar(p, starts, prefix);
  const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  auto report = [&](uint32_t pos, uint32_t code, uint32_t index) {
    atomicMin(first + shard_slot(p.whole, p.whole ? 0u : doc_of(p.a, pos), p.owned), (static_cast<unsigned long long>(index) << 8) | code);
  };
  for (uint32_t t = blockIdx.x * kWarps + w; t < tiles; t += gridDim.x * kWarps) {
    load_tile<kItems>(g, sm[w], lane, t * kTile, h);
    tile_check<kItems>(g, sm[w], lane, t * kTile, t, report, h);
  }
}

// the results of the documents that start here but the last (whose end is known after the result round), or with
// bad = 1 every result {UNEXPECTED_ERROR, none}
__global__ void __launch_bounds__(256) gram_shard_result_kernel(ShardPass p, const unsigned long long *first, uint32_t *tally, int bad) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= p.owned || (!bad && d + 1 >= p.owned)) return;
  sjb200_sharded_document_error_t r{0, 0, 0};
  if (bad) {
    r.error = int32_t(kUnexpected);
    r.index = ~0ull;
  } else {
    shard_doc_result(first[d], p.tokens_before, p.a.docs[d + 1].index, &r.error, &r.index);
    if (r.error != 0) {
      atomicAdd(tally + 1, 1u);
      atomicMin(tally + 2, d);
    }
  }
  p.out[d] = r;
}

// result round: the tally words of sjb200_params.h into every window, one thread per rank
__global__ void gram_shard_post_result_kernel(const unsigned long long *first, const uint32_t *tally, uint32_t owned, uint64_t tokens_before,
                                              const __grid_constant__ Xchg x, size_t at) {
  const uint32_t r = threadIdx.x;
  if (r >= x.nranks) return;
  uint32_t w[kGramResWords];
  shard_result_words(first, owned, tokens_before, tally[1], tally[2], w);
  for (int k = 0; k < kGramResWords; k++) store_tagged(x, r, at + kGramResAt + k, w[k]);
}

__global__ void gram_shard_store_kernel(sjb200_sharded_document_error_t *out, int32_t error, uint64_t index) {
  *out = sjb200_sharded_document_error_t{error, 0, index};
}

}  // namespace

size_t shard_scratch_words(uint32_t n, uint32_t ndocs, uint32_t max_depth) {
  const size_t stride = 2 + (max_depth + 31) / 32;
  uint32_t count[8];
  const int L = tree_levels((n + kTile - 1) / kTile, count, 8);
  size_t recs = 1;  // the incoming record
  for (int l = 0; l < L; l++) recs += count[l];
  return 2 * (size_t(ndocs ? ndocs : 1) + 1) + 4 + (size_t(n) + 31) / 32 + 1 + recs * stride;
}

cudaError_t launch_shard_edges(const GrammarArgs &a, bool whole, uint32_t max_depth_word, bool failed, uint32_t *scratch, const Xchg &rec, size_t at,
                               cudaStream_t st, int *launches) {
  *launches = 0;
  if (!failed) {
    const ShardScratch s = shard_layout(scratch, a.n, a.ndocs, a.max_depth);
    const uint32_t init[4] = {0, 0, kNone, 0};
    cudaError_t e = cudaMemsetAsync(s.first, 0xFF, sizeof(unsigned long long) * (size_t(a.ndocs ? a.ndocs : 1) + 1), st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(s.tally, init, sizeof(init), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(s.starts, 0, sizeof(uint32_t) * ((size_t(a.n) + 31) / 32 + 1), st);
    if (e != cudaSuccess) return e;
    if (!whole && a.docs && a.ndocs) {
      gram_shard_starts_kernel<<<(a.ndocs + 255) / 256, 256, 0, st>>>(a, s.starts, s.tally);
      ++*launches;
    }
    gram_shard_edges_kernel<<<1, 32, 0, st>>>(a, whole, max_depth_word, 0, s.tally, rec, at);
  } else {
    gram_shard_edges_kernel<<<1, 32, 0, st>>>(a, whole, max_depth_word, 1, nullptr, rec, at);
  }
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_shard_records(const ShardPass &p, const ShardHalo &h, bool root, uint32_t *scratch, int sm_count, const Xchg &x, size_t at,
                                 cudaStream_t st, int *launches) {
  const ShardScratch s = shard_layout(scratch, p.a.n, p.a.ndocs, p.a.max_depth);
  const uint32_t words = (p.a.max_depth + 31) / 32;
  const uint32_t tiles = (p.a.n + kTile - 1) / kTile;
  *launches = 1;
  if (tiles) {
    if (root) {
      gram_shard_root_kernel<<<1, 1, 0, st>>>(s.starts);
      ++*launches;
    }
    gram_shard_record_kernel<<<grid_for(tiles, kWarps, sm_count, 16), kWarps * 32, 0, st>>>(p, h, s.starts, s.level[0], tiles);
    for (int l = 0; l + 1 < s.L; l++)
      gram_up_kernel<<<grid_for((s.count[l] + 31) / 32, kWarps, sm_count, 16), kWarps * 32, 0, st>>>(s.level[l], s.count[l], s.level[l + 1], words);
    *launches += s.L;
  }
  gram_shard_post_record_kernel<<<1, 32, 0, st>>>(tiles ? s.level[s.L - 1] : nullptr, words, x, at);
  return cudaGetLastError();
}

cudaError_t launch_shard_check(const ShardPass &p, const ShardHalo &h, uint32_t *scratch, const unsigned long long *win, int sm_count, const Xchg &x,
                               size_t at, cudaStream_t st, int *launches) {
  const ShardScratch s = shard_layout(scratch, p.a.n, p.a.ndocs, p.a.max_depth);
  const uint32_t words = (p.a.max_depth + 31) / 32;
  const uint32_t tiles = (p.a.n + kTile - 1) / kTile;
  *launches = 2;
  if (tiles) {
    gram_shard_incoming_kernel<<<1, 32, 0, st>>>(win, x.rank, words, s.incoming);
    for (int l = s.L - 1; l >= 0; l--)
      gram_down_kernel<<<grid_for((s.count[l] + 31) / 32, kWarps, sm_count, 16), kWarps * 32, 0, st>>>(s.level[l], s.count[l],
                                                                                                       l + 1 < s.L ? s.level[l + 1] : s.incoming, words);
    gram_shard_check_kernel<<<grid_for(tiles, kWarps, sm_count, 16), kWarps * 32, 0, st>>>(p, h, s.starts, s.level[0], s.first, tiles);
    *launches += s.L + 2;
  }
  if (p.owned > 1) {
    gram_shard_result_kernel<<<(p.owned + 255) / 256, 256, 0, st>>>(p, s.first, s.tally, 0);
    ++*launches;
  }
  gram_shard_post_result_kernel<<<1, 32, 0, st>>>(s.first, s.tally, p.owned, p.tokens_before, x, at);
  return cudaGetLastError();
}

cudaError_t launch_shard_fill_bad(const ShardPass &p, cudaStream_t st) {
  if (p.owned) gram_shard_result_kernel<<<(p.owned + 255) / 256, 256, 0, st>>>(p, nullptr, nullptr, 1);
  return cudaGetLastError();
}

cudaError_t launch_shard_store(sjb200_sharded_document_error_t *out, int32_t error, uint64_t index, cudaStream_t st) {
  gram_shard_store_kernel<<<1, 1, 0, st>>>(out, error, index);
  return cudaGetLastError();
}

}  // namespace gram
}  // namespace sjb200
