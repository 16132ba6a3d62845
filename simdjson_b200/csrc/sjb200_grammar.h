// sjb200_grammar.h -- launcher of sjb200_grammar.cu (the nesting grammar of stage 2, sjb200_document_errors_dev)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_docs.h"
#include "sjb200_grammar.cuh"

namespace sjb200 {
namespace gram {

// structurals per tile: 32 lanes x kItems (DESIGN.md section 4.7)
constexpr int kItems = 32;
constexpr uint32_t kTile = 32u * kItems;

struct GrammarArgs {
  const uint8_t *type;
  const uint64_t *payload;
  uint32_t n;
  const sjb200_doc_boundary_t *docs;  // null: one document [0, n)
  uint32_t ndocs;
  uint32_t max_depth;                 // 1 .. kMaxDepth
  DocError *out;                      // [docs ? ndocs : 1]
};

// words of device scratch a call needs
size_t grammar_scratch_words(uint32_t n, uint32_t ndocs, uint32_t max_depth);
// Every launch on s, no synchronisation (*launches: the kernels enqueued).  summary (3 words of device memory): [0] != 0
// when the table is bad, [1] the documents in error, [2] the first of them (0xFFFFFFFF: none).
cudaError_t launch_document_errors(const GrammarArgs &a, uint32_t *scratch, uint32_t *summary, int sm_count, cudaStream_t s, int *launches);


// ---- one rank's part of a sharded pass (sjb200_document_errors_sharded, sjb200_comm.cu).  The scratch of a pass:
// first[D + 1] (the last: the leading segment's), a tally of 4 words, the start bitmap, the fold tree, the incoming record.
struct sjb200_sharded_document_error_t;
struct ShardPass {
  GrammarArgs a;                    // docs: the rank's table (whole mode: null); out unused
  bool whole;
  uint32_t owned;                   // documents that start here: ndocs, or whole mode 1 on rank 0 and 0 elsewhere
  uint64_t tokens_before;
  sjb200_sharded_document_error_t *out;
};
struct sjb200_sharded_document_error_t {
  int32_t error;
  uint32_t reserved;
  uint64_t index;
};
size_t shard_scratch_words(uint32_t n, uint32_t ndocs, uint32_t max_depth);
// enqueue: the table's check and start bitmap, then the edge words and the pass's round-0 record into every window
cudaError_t launch_shard_edges(const GrammarArgs &a, bool whole, uint32_t max_depth_word, bool failed, uint32_t *scratch, const Xchg &rec, size_t at,
                               cudaStream_t s, int *launches);
// record round: pass A with the halo, the fold tree up, its top record into every window (2 + words words at `at`)
cudaError_t launch_shard_records(const ShardPass &p, const ShardHalo &h, bool root, uint32_t *scratch, int sm_count, const Xchg &x, size_t at,
                                 cudaStream_t s, int *launches);
// result round: the incoming record from the earlier ranks' (window words at `win`, kGramWords apart), the fold tree down,
// pass C, this rank's results but its last document's, and its tally words into every window at `at`
cudaError_t launch_shard_check(const ShardPass &p, const ShardHalo &h, uint32_t *scratch, const unsigned long long *win, int sm_count, const Xchg &x,
                               size_t at, cudaStream_t s, int *launches);
// every result {UNEXPECTED_ERROR, none} (a bad table somewhere), or one result
cudaError_t launch_shard_fill_bad(const ShardPass &p, cudaStream_t s);
cudaError_t launch_shard_store(sjb200_sharded_document_error_t *out, int32_t error, uint64_t index, cudaStream_t s);

}  // namespace gram
}  // namespace sjb200
