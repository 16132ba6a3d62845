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

}  // namespace

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
