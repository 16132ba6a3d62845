// sjb200_tape.h -- launcher of sjb200_tape.cu (stage-2-lite on the device, SURVEY.md section 8(f) row 4)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_params.h"

namespace sjb200 {

struct TokenTotals {
  unsigned long long string_bytes;  // bytes of string_buf the document's strings need (records of valid strings)
  unsigned long long first_error;   // (structural index << 8) | error_code of the first token in error, ~0 when none
  uint32_t n_strings;
  uint32_t reserved;
};

// A sharded tokens pass (sjb200_comm): where tile_scan_kernel stores the shard's record (window slot xchg.slot, kind
// kTokens) and its summary (xchg_summary_at(seq, rank)) in every rank's window, and what they carry besides the totals.
// xchg.nranks == 0: no exchange.
struct TokXchg {
  Xchg xchg;
  uint32_t state_in;   // the scanner state the caller says the shard starts in (0: a clean cut)
  uint32_t n;
  uint64_t len;
  uint64_t capacity;   // this rank's string buffer
};

// tile_scan_kernel, the scan of the tokens' tile sums, for another per-tile quantity (sjb200_column_dev): tile_sums[ntiles] become
// their exclusive prefix sums, tot->string_bytes their total and tot->n_strings the total of tile_counts[ntiles].  One CTA.
cudaError_t launch_tile_scan(unsigned long long *tile_sums, const uint32_t *tile_counts, uint32_t ntiles, TokenTotals *tot, cudaStream_t stream);

size_t tokens_scratch_bytes(uint32_t n);
// type[n], payload[n], strbuf[strbuf_capacity]: device memory; scratch: tokens_scratch_bytes(n) bytes, 8-byte aligned;
// stage: 1 = tiles staged through shared memory (the product path), 0 = every thread reads / writes global memory (kept as
// the A/B baseline of the staging, option tok_stage).  xchg: a sharded pass's exchange, fused into the scan of the tile
// sums (null: none)
cudaError_t launch_tokens(const uint8_t *buf, uint64_t len, const uint32_t *idx, uint32_t n, uint8_t *type, uint64_t *payload, uint8_t *strbuf,
                          uint64_t strbuf_capacity, void *scratch, TokenTotals *tot_dev, int stage, cudaStream_t stream, const TokXchg *xchg = nullptr);

}  // namespace sjb200
