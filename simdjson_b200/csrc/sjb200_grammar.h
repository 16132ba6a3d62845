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

}  // namespace gram
}  // namespace sjb200
