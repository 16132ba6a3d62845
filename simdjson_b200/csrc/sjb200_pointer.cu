// sjb200_pointer.cu -- JSON Pointer lookup on the device for every document of a stream (sjb200_at_pointer_dev): the
// token-error pass and the two walks of sjb200_pointer.cuh, one warp or one CTA per (document, pointer).
#include "sjb200_pointer.h"

namespace sjb200 {
namespace ptr {
namespace {

// the document's structurals [*start, *end); false: the table entry is not ascending or not below n
__device__ __forceinline__ bool doc_span(const PtrLaunch &a, uint32_t d, uint32_t *start, uint32_t *end) {
  if (!a.docs) {
    *start = 0;
    *end = a.n;
    return a.n > 0;
  }
  const uint32_t s = a.docs[d].index;
  if (s >= a.n || (d > 0 && a.docs[d - 1].index >= s)) return false;
  uint32_t e = a.n;
  if (d + 1 < a.ndocs) {
    const uint32_t nx = a.docs[d + 1].index;
    if (nx > s && nx < a.n) e = nx;
  }
  *start = s;
  *end = e;
  return true;
}

// the last document whose start is <= k (kNone: before the first); on an ascending table that is k's document
__device__ __forceinline__ uint32_t doc_of(const PtrLaunch &a, uint32_t k) {
  if (!a.docs) return 0;
  uint32_t lo = 0, hi = a.ndocs;  // answer in [lo - 1, hi)
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (a.docs[mid].index <= k) lo = mid + 1; else hi = mid;
  }
  return lo == 0 ? kNone : lo - 1;
}

// One read of the token types: the first token in error of each document (atomicMin), and the list of documents longer
// than the warp walk's limit.  first_err must hold kNone and *long_count 0.
__global__ void __launch_bounds__(256) ptr_prep_kernel(PtrLaunch a) {
  const uint64_t D = a.docs ? a.ndocs : 1;
  const uint64_t N = a.n > D ? a.n : D;
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    if (i < a.n && a.w.type[i] == 0) {
      const uint32_t d = doc_of(a, uint32_t(i));
      if (d != kNone) atomicMin(a.first_err + d, uint32_t(i));
    }
    uint32_t s, e;
    if (i < D && doc_span(a, uint32_t(i), &s, &e) && e - s > kCtaMinStructurals) a.long_docs[atomicAdd(a.long_count, 1u)] = uint32_t(i);
  }
}

// The result of a document that needs no walk: a bad table entry or a token in error.  false: it needs one.
__device__ __forceinline__ bool settled(const PtrLaunch &a, uint32_t d, uint32_t *s, uint32_t *e, int32_t *err, uint32_t *idx) {
  if (!doc_span(a, d, s, e)) {
    *err = kUnexpectedError;
    *idx = kNone;
    return true;
  }
  const uint32_t fe = a.first_err[d];
  if (fe == kNone) return false;
  *err = int32_t(a.w.payload[fe]);
  *idx = fe;
  return true;
}

// one warp per (document, pointer), pointer-major; documents over kCtaMinStructurals are left to ptr_cta_kernel
__global__ void __launch_bounds__(256) ptr_warp_kernel(PtrLaunch a) {
  const uint64_t D = a.docs ? a.ndocs : 1;
  const uint64_t jobs = D * a.npointers;
  const uint64_t stride = (uint64_t(gridDim.x) * blockDim.x) >> 5;
  WarpGroup g{threadIdx.x & 31u};
  for (uint64_t j = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; j < jobs; j += stride) {
    const uint32_t p = uint32_t(j / D), d = uint32_t(j % D);
    uint32_t s, e, idx;
    int32_t err;
    if (!settled(a, d, &s, &e, &err, &idx)) {
      if (e - s > kCtaMinStructurals) continue;
      idx = walk_pointer<WarpGroup, 1>(g, a.w, a.headers[p], s, e, &err);
    }
    if (g.lane == 0) a.out[j] = PtrResult{err, idx};
  }
}

// one CTA per (long document, pointer)
__global__ void __launch_bounds__(kCtaWarps * 32) ptr_cta_kernel(PtrLaunch a) {
  __shared__ CtaSmem<kCtaWarps> sm;
  CtaGroup<kCtaWarps> g{threadIdx.x, &sm};
  const uint64_t D = a.docs ? a.ndocs : 1;
  const uint64_t jobs = uint64_t(*a.long_count) * a.npointers;
  for (uint64_t j = blockIdx.x; j < jobs; j += gridDim.x) {
    const uint32_t d = a.long_docs[j / a.npointers], p = uint32_t(j % a.npointers);
    uint32_t s, e, idx;
    int32_t err;
    if (settled(a, d, &s, &e, &err, &idx)) continue;  // written by ptr_warp_kernel
    idx = walk_pointer<CtaGroup<kCtaWarps>, kCtaItems>(g, a.w, a.headers[p], s, e, &err);
    if (threadIdx.x == 0) a.out[uint64_t(p) * D + d] = PtrResult{err, idx};
  }
}

// =============================================================================== one rank of a sharded pass
// scratch: [0] long documents, [1] the table is bad, [2] the leading segment's first token in error, [3] walks handed
// over in the current step, [4, 4 + D) each document's first token in error, [4 + D, 4 + 2 D) the long documents
constexpr uint32_t kShardHead = 4;
__device__ __forceinline__ uint32_t *shard_forwarded(uint32_t *scratch) { return scratch + 3; }

__device__ __forceinline__ uint32_t shard_docs(const PtrShard &s) { return s.a.docs ? s.a.ndocs : 1u; }
// the end of the leading segment: the table's first entry, or n
__device__ __forceinline__ uint32_t shard_lead_end(const PtrLaunch &a) { return a.docs ? a.docs[0].index : a.n; }

// the table's check, each document's and the leading segment's first token in error, and the long documents
__global__ void __launch_bounds__(256) ptr_shard_prep_kernel(PtrShard s) {
  const PtrLaunch &a = s.a;
  uint32_t *first_err = s.scratch + kShardHead, *long_docs = first_err + shard_docs(s);
  const uint64_t D = shard_docs(s);
  const uint64_t N = a.n > D ? a.n : D;
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  const uint32_t lead_end = shard_lead_end(a);
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    if (i < a.n && a.w.type[i] == 0) {
      const uint32_t d = doc_of(a, uint32_t(i));
      if (d != kNone) atomicMin(first_err + d, uint32_t(i));
      if (i < lead_end) atomicMin(s.scratch + 2, uint32_t(i));
    }
    if (i < D) {
      uint32_t b, e;
      if (!doc_span(a, uint32_t(i), &b, &e)) {
        if (a.docs) atomicOr(s.scratch + 1, 1u);
      } else if (e - b > kCtaMinStructurals) {
        long_docs[atomicAdd(s.scratch, 1u)] = uint32_t(i);
      }
    }
  }
}

__device__ __forceinline__ void store_tagged(const Xchg &x, uint32_t r, size_t at, uint32_t w) {
  sj_st_sys_u64(x.peer[r] + at, (static_cast<unsigned long long>(x.seq) << 32) | w);
}

// the edge words and the round-0 record, one thread per rank
__global__ void ptr_shard_edges_kernel(PtrShard s, uint32_t flags, uint64_t hash, const __grid_constant__ Xchg x, size_t at) {
  const uint32_t r = threadIdx.x;
  if (r >= x.nranks) return;
  const bool failed = flags & kPtrEdgeFailed;
  const uint32_t n = s.a.n;
  const uint32_t lead = failed ? kNone : s.scratch[2];
  uint32_t w[kPtrEdgeWords];
  w[0] = n;
  w[1] = s.a.docs ? s.a.ndocs : 0u;
  w[2] = flags | (!failed && s.scratch[1] ? uint32_t(kPtrEdgeBadTable) : 0u);
  w[3] = s.a.npointers;
  w[4] = uint32_t(hash);
  w[5] = uint32_t(hash >> 32);
  w[6] = (n && !failed) ? uint32_t(s.a.w.type[0]) | (uint32_t(s.a.w.type[n - 1]) << 8) : 0xFFFFu;
  w[7] = failed ? n : shard_lead_end(s.a);
  w[8] = lead;
  w[9] = lead == kNone ? 0u : uint32_t(s.a.w.payload[lead]) & 0xFFu;
  for (int k = 0; k < kPtrEdgeWords; k++) store_tagged(x, r, at + size_t(x.rank) * kPtrEdgeWords + k, w[k]);
  unsigned long long *rec = x.peer[r] + (size_t(x.slot) * kMaxRanks + x.rank) * 2;
  sj_st_sys_u64(rec, xchg_word0(x.seq, n));
  sj_st_sys_u64(rec + 1, xchg_word1(x.seq, 0, 0, failed ? uint32_t(kFlagInternal) : 0u, kPointer));
}

// a finished walk: into this rank's out (res null: the document is this rank's, number d) or the owner's result area
__device__ __forceinline__ void shard_put(const PtrShard &s, uint32_t p, uint32_t d, unsigned long long *res, int32_t err, uint64_t index) {
  if (res) {
    sj_st_sys_u64(res + 2 * size_t(p), (static_cast<unsigned long long>(s.seq) << 32) | uint32_t(err));
    sj_st_sys_u64(res + 2 * size_t(p) + 1, index);
  } else {
    s.out[uint64_t(p) * s.owned + d] = ShardPtrResult{err, 0, index};
  }
}

// the walk of pointer p over the piece [.., end) of this rank from `at`; the group's rank 0 reports
template <class G, int ITEMS>
__device__ __forceinline__ void shard_walk(G &g, const PtrShard &s, uint32_t p, WalkAt at, uint32_t end, uint32_t d, unsigned long long *res) {
  int32_t err;
  WalkAt susp;
  const uint32_t v = walk_from<G, ITEMS>(g, s.a.w, s.a.headers[p], at, end, piece_cut(s.v, end), &err, &susp);
  if (g.rank() != 0) return;
  if (v == kSuspend) {
    unsigned long long w0, w1;
    pack_walk(susp, s.seq, s.step, &w0, &w1);
    sj_st_sys_u64(s.next_rec + 2 * size_t(p), w0);
    sj_st_sys_u64(s.next_rec + 2 * size_t(p) + 1, w1);
    atomicAdd(shard_forwarded(s.scratch), 1u);
    return;
  }
  shard_put(s, p, d, res, err, v == kNone ? ~0ull : s.tokens_before + v);
}

// a document that needs no walk: a token in error in its piece here, or (the tail document) in its later pieces
__device__ __forceinline__ bool shard_settled(const PtrShard &s, uint32_t d, uint32_t e, int32_t *err, uint64_t *index) {
  const uint32_t fe = s.scratch[kShardHead + d];
  if (fe != kNone) {
    *err = int32_t(s.a.w.payload[fe]);
    *index = s.tokens_before + fe;
    return true;
  }
  if (e == s.a.n && s.tail_err != 0) {
    *err = s.tail_err;
    *index = s.tail_err_index;
    return true;
  }
  return false;
}

// step 0, one warp per (document starting here, pointer); documents over kCtaMinStructurals are left to the CTA kernel
__global__ void __launch_bounds__(256) ptr_shard_warp_kernel(PtrShard s) {
  const uint64_t D = shard_docs(s);
  const uint64_t jobs = D * s.a.npointers;
  const uint64_t stride = (uint64_t(gridDim.x) * blockDim.x) >> 5;
  WarpGroup g{threadIdx.x & 31u};
  for (uint64_t j = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; j < jobs; j += stride) {
    const uint32_t p = uint32_t(j / D), d = uint32_t(j % D);
    uint32_t b, e;
    doc_span(s.a, d, &b, &e);  // (a bad table never gets here)
    unsigned long long *res = e == s.a.n ? s.tail_res : nullptr;
    int32_t err;
    uint64_t index;
    if (shard_settled(s, d, e, &err, &index)) {
      if (g.lane == 0) shard_put(s, p, d, res, err, index);
      continue;
    }
    if (e - b > kCtaMinStructurals) continue;
    shard_walk<WarpGroup, 1>(g, s, p, WalkAt{0, b, 0, 0, 0, 0}, e, d, res);
  }
}

// step 0, one CTA per (long document starting here, pointer)
__global__ void __launch_bounds__(kCtaWarps * 32) ptr_shard_cta_kernel(PtrShard s) {
  __shared__ CtaSmem<kCtaWarps> sm;
  CtaGroup<kCtaWarps> g{threadIdx.x, &sm};
  const uint32_t *long_docs = s.scratch + kShardHead + shard_docs(s);
  const uint64_t jobs = uint64_t(s.scratch[0]) * s.a.npointers;
  for (uint64_t j = blockIdx.x; j < jobs; j += gridDim.x) {
    const uint32_t d = long_docs[j / s.a.npointers], p = uint32_t(j % s.a.npointers);
    uint32_t b, e;
    doc_span(s.a, d, &b, &e);
    int32_t err;
    uint64_t index;
    if (shard_settled(s, d, e, &err, &index)) continue;  // written by the warp kernel
    shard_walk<CtaGroup<kCtaWarps>, kCtaItems>(g, s, p, WalkAt{0, b, 0, 0, 0, 0}, e, d, e == s.a.n ? s.tail_res : nullptr);
  }
}

// step > 0: the walks handed over in the previous step, resumed over the leading segment; one group per pointer
template <class G, int ITEMS>
__device__ __forceinline__ void shard_resume(G &g, const PtrShard &s, uint32_t p) {
  WalkAt at;
  if (!unpack_walk(s.rec_in[2 * size_t(p)], s.rec_in[2 * size_t(p) + 1], s.seq, s.step - 1, &at)) return;
  shard_walk<G, ITEMS>(g, s, p, at, s.lead_end, 0, s.lead_res);
}

// (at most kPtrMaxPointers groups: one launch covers them)
__global__ void __launch_bounds__(256) ptr_shard_resume_warp_kernel(PtrShard s) {
  WarpGroup g{threadIdx.x & 31u};
  const uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (p < s.a.npointers) shard_resume<WarpGroup, 1>(g, s, p);
}

// (a register cap instead of launch bounds: with the bounds ptxas stops at 48 registers and spills)
__global__ void __maxnreg__(64) ptr_shard_resume_cta_kernel(PtrShard s) {
  __shared__ CtaSmem<kCtaWarps> sm;
  CtaGroup<kCtaWarps> g{threadIdx.x, &sm};
  shard_resume<CtaGroup<kCtaWarps>, kCtaItems>(g, s, blockIdx.x);
}

// the count of a step into every rank's window, one thread per rank; the counter starts again from 0
__global__ void ptr_shard_count_kernel(uint32_t *scratch, const __grid_constant__ Xchg x, size_t at, uint32_t step) {
  const uint32_t r = threadIdx.x;
  const uint32_t c = *shard_forwarded(scratch);
  __syncthreads();
  if (r < x.nranks) store_tagged(x, r, at + kPtrCountAt + size_t(x.rank) * kMaxRanks + step, c);
  if (r == 0) *shard_forwarded(scratch) = 0;
}

__global__ void __launch_bounds__(256) ptr_shard_scatter_kernel(const unsigned long long *res, uint32_t seq, ShardPtrResult *out, uint32_t np, uint32_t owned) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= np) return;
  const unsigned long long w0 = res[2 * size_t(p)];
  if (uint32_t(w0 >> 32) == seq) out[uint64_t(p) * owned + owned - 1] = ShardPtrResult{int32_t(uint32_t(w0)), 0, res[2 * size_t(p) + 1]};
}

__global__ void __launch_bounds__(256) ptr_shard_fill_kernel(ShardPtrResult *out, uint64_t count, int32_t error) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += uint64_t(gridDim.x) * blockDim.x) out[i] = ShardPtrResult{error, 0, ~0ull};
}

unsigned grid_of(uint64_t blocks, int sm_count, int per_sm) { return unsigned(blocks < uint64_t(sm_count) * per_sm ? (blocks ? blocks : 1) : uint64_t(sm_count) * per_sm); }

}  // namespace

size_t shard_scratch_words(uint32_t ndocs) { return kShardHead + 2 * size_t(ndocs ? ndocs : 1); }

cudaError_t launch_shard_edges(const PtrShard &s, uint32_t flags, uint64_t hash, const Xchg &x, size_t at, int sm_count, cudaStream_t st, int *launches) {
  *launches = 1;
  if (!(flags & kPtrEdgeFailed)) {
    const uint32_t D = s.a.docs ? s.a.ndocs : 1;
    const uint32_t init[kShardHead] = {0, 0, kNone, 0};
    cudaError_t e = cudaMemcpyAsync(s.scratch, init, sizeof(init), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(s.scratch + kShardHead, 0xFF, sizeof(uint32_t) * size_t(D), st);
    if (e != cudaSuccess) return e;
    const uint64_t N = s.a.n > D ? s.a.n : D;
    ptr_shard_prep_kernel<<<grid_of((N + 255) / 256, sm_count, 8), 256, 0, st>>>(s);
    ++*launches;
  }
  ptr_shard_edges_kernel<<<1, 32, 0, st>>>(s, flags, hash, x, at);
  return cudaGetLastError();
}

cudaError_t launch_shard_walks(const PtrShard &s, int sm_count, cudaStream_t st, int *launches) {
  *launches = 0;
  if (!s.walks) return cudaSuccess;
  const uint64_t D = s.a.docs ? s.a.ndocs : 1;
  ptr_shard_warp_kernel<<<grid_of((D * s.a.npointers + 7) / 8, sm_count, 16), 256, 0, st>>>(s);
  ptr_shard_cta_kernel<<<unsigned(sm_count) * 2, kCtaWarps * 32, 0, st>>>(s);
  *launches = 2;
  return cudaGetLastError();
}

cudaError_t launch_shard_resume(const PtrShard &s, bool cta, cudaStream_t st) {
  if (!s.a.npointers) return cudaSuccess;
  if (cta)
    ptr_shard_resume_cta_kernel<<<s.a.npointers, kCtaWarps * 32, 0, st>>>(s);
  else
    ptr_shard_resume_warp_kernel<<<(s.a.npointers + 7) / 8, 256, 0, st>>>(s);
  return cudaGetLastError();
}

cudaError_t launch_shard_post_count(uint32_t *scratch, const Xchg &x, size_t at, uint32_t step, cudaStream_t st) {
  ptr_shard_count_kernel<<<1, 32, 0, st>>>(scratch, x, at, step);
  return cudaGetLastError();
}

cudaError_t launch_shard_scatter(const unsigned long long *res, uint32_t seq, ShardPtrResult *out, uint32_t npointers, uint32_t owned, cudaStream_t st) {
  if (npointers && owned) ptr_shard_scatter_kernel<<<(npointers + 255) / 256, 256, 0, st>>>(res, seq, out, npointers, owned);
  return cudaGetLastError();
}

cudaError_t launch_shard_fill(ShardPtrResult *out, uint64_t count, int32_t error, int sm_count, cudaStream_t st) {
  if (count) ptr_shard_fill_kernel<<<grid_of((count + 255) / 256, sm_count, 8), 256, 0, st>>>(out, count, error);
  return cudaGetLastError();
}

size_t pointer_scratch_words(uint32_t ndocs) { return 1 + 2 * size_t(ndocs); }

cudaError_t launch_at_pointer(const PtrLaunch &args, uint32_t *scratch, int sm_count, cudaStream_t s) {
  PtrLaunch a = args;
  const uint32_t D = a.docs ? a.ndocs : 1;
  a.long_count = scratch;
  a.first_err = scratch + 1;
  a.long_docs = scratch + 1 + D;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(uint32_t), s);
  if (e == cudaSuccess) e = cudaMemsetAsync(a.first_err, 0xFF, sizeof(uint32_t) * size_t(D), s);
  if (e != cudaSuccess) return e;
  const uint64_t N = a.n > D ? a.n : D;
  const uint64_t prep_blocks = (N + 255) / 256;
  ptr_prep_kernel<<<unsigned(prep_blocks < uint64_t(sm_count) * 8 ? prep_blocks : uint64_t(sm_count) * 8), 256, 0, s>>>(a);
  const uint64_t warp_blocks = (uint64_t(D) * a.npointers + 7) / 8;
  ptr_warp_kernel<<<unsigned(warp_blocks < uint64_t(sm_count) * 16 ? warp_blocks : uint64_t(sm_count) * 16), 256, 0, s>>>(a);
  ptr_cta_kernel<<<unsigned(sm_count) * 2, kCtaWarps * 32, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace ptr
}  // namespace sjb200
