// sjb200_grammar.cu -- the nesting grammar of stage 2 for every document of a stream (sjb200_document_errors_dev): the
// tile routines of sjb200_grammar.cuh as sm_90a kernels.  Launch order on one stream: the document-start bitmap, the
// tile records (pass A), the fold tree up and down (pass B), the judgement of every structural (pass C), the results.
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

}  // namespace gram
}  // namespace sjb200
