// sjb200_pointer.h -- launcher of sjb200_pointer.cu (JSON Pointer lookup, sjb200_at_pointer_dev)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_docs.h"
#include "sjb200_pointer.cuh"

namespace sjb200 {
namespace ptr {

// A document of more structurals than this is walked by a CTA of kCtaWarps warps, kCtaItems structurals per thread per
// step; one of at most this many by a warp, one structural per lane per step (DESIGN.md section 4.6).
#ifndef SJB200_POINTER_CTA_MIN
#define SJB200_POINTER_CTA_MIN 4096
#endif
constexpr uint32_t kCtaMinStructurals = SJB200_POINTER_CTA_MIN;
constexpr unsigned kCtaWarps = 8;
constexpr int kCtaItems = 8;

struct PtrResult {  // sjb200_pointer_result
  int32_t error;
  uint32_t index;
};

struct PtrLaunch {
  Walk w;
  uint32_t n;
  const sjb200_doc_boundary_t *docs;  // null: one document [0, n)
  uint32_t ndocs;
  const PtrHeader *headers;
  uint32_t npointers;
  PtrResult *out;  // [npointers][docs ? ndocs : 1]
  // scratch, set by launch_at_pointer
  uint32_t *long_count, *first_err, *long_docs;
};

// ---- one rank of a sharded pass (sjb200_at_pointer_sharded)
struct ShardPtrResult {  // sjb200_sharded_pointer_result
  int32_t error;
  uint32_t reserved;
  uint64_t index;
};

struct PtrShard {
  PtrLaunch a;                       // this rank's tokens, table (null in whole mode) and pointers; a.out is unused
  ShardView v;
  ShardPtrResult *out;               // [npointers][owned]
  uint64_t tokens_before;
  uint32_t owned;                    // results this rank writes (whole mode: 1 on rank 0)
  uint32_t walks;                    // documents walked here from their roots (whole mode: 1 on the first holder)
  uint32_t lead_end;                 // (finish) the table's first entry, or n: this rank's leading segment is [0, lead_end)
  int32_t tail_err;                  // the first token in error of the tail document's pieces on later ranks (0: none)
  uint64_t tail_err_index;           // its global index
  unsigned long long *next_rec;      // the next holder's record buffer of this step (null: none)
  unsigned long long *tail_res;      // result area of the owner of the document holding n - 1; null: this rank's out
  unsigned long long *lead_res;      // that of the owner of the document of the leading segment
  const unsigned long long *rec_in;  // this rank's record buffer of the previous step
  uint32_t seq, step;
  uint32_t *scratch;                 // shard_scratch_words(ndocs) words, the layout of sjb200_pointer.cu
};

// scratch words of a rank's pass (kept from enqueue to finish)
size_t shard_scratch_words(uint32_t ndocs);
// enqueue: the first token in error of each document and of the leading segment, the table's check, then the edge
// words (sjb200_params.h) and the pass's round-0 record into every rank's window.  failed: publish only, flagged.
cudaError_t launch_shard_edges(const PtrShard &s, uint32_t flags, uint64_t hash, const Xchg &x, size_t at, int sm_count, cudaStream_t st, int *launches);
// step 0: the walks of the documents that start here (warp and CTA walks as launch_at_pointer)
cudaError_t launch_shard_walks(const PtrShard &s, int sm_count, cudaStream_t st, int *launches);
// step > 0: resume the walks handed over in the previous step, by warps (cta = 0) or CTAs
cudaError_t launch_shard_resume(const PtrShard &s, bool cta, cudaStream_t st);
// the walks this rank handed over in step `step` into every rank's count words (and the counter back to 0)
cudaError_t launch_shard_post_count(uint32_t *scratch, const Xchg &x, size_t at, uint32_t step, cudaStream_t st);
// the results of this rank's last document that came back from later ranks (tagged seq in res) into out[p][owned - 1]
cudaError_t launch_shard_scatter(const unsigned long long *res, uint32_t seq, ShardPtrResult *out, uint32_t npointers, uint32_t owned, cudaStream_t st);
// every result {error, UINT64_MAX}
cudaError_t launch_shard_fill(ShardPtrResult *out, uint64_t count, int32_t error, int sm_count, cudaStream_t st);

size_t pointer_scratch_words(uint32_t ndocs);
// scratch: pointer_scratch_words(ndocs) words of device memory.  Three launches on s, no synchronisation.
cudaError_t launch_at_pointer(const PtrLaunch &a, uint32_t *scratch, int sm_count, cudaStream_t s);

}  // namespace ptr
}  // namespace sjb200
