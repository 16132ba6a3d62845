// sjb200_docs.h -- launchers of sjb200_docs.cu (device-side epilogue of streaming scans, document boundary table)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_params.h"

namespace sjb200 {

// what the streaming branches of finish() produce (json_structural_indexer.h L249-343)
struct StreamFinish {
  int32_t err;         // simdjson::error_code
  uint32_t n;          // n_structural_indexes (valid when n_written)
  uint32_t n_written;  // 0: the call returned before touching n (UNESCAPED_CHARS / internal error)
  uint32_t reserved;
};
// same layout as sjb200_doc_boundary (include/sjb200.h)
struct sjb200_doc_boundary_t {
  uint32_t index;  // structural index at which a document starts
  uint32_t byte;   // = structural_indexes[index]
};

// modes 1 / 2 (streaming_partial / streaming_final) behind a device-resident scan whose result block is `carry`
cudaError_t launch_stream_finish(const uint8_t *buf, uint32_t *idx, const Carry *carry, uint32_t len, int mode, StreamFinish *out_dev, StreamFinish *out_host,
                                 cudaStream_t stream);
// modes 3..6 (RS-delimited / comma-delimited streams): filter the device-resident index array in place and run the
// rest of finish(); n = structurals to consider (host-known), scratch: filter_scratch_words(n) uint32 words
size_t filter_scratch_words(uint32_t n);
cudaError_t launch_stream_filter(const uint8_t *buf, uint32_t len, uint32_t *idx, uint32_t n, int mode, uint32_t flags, uint32_t *scratch, StreamFinish *out_dev,
                                 StreamFinish *out_host, cudaStream_t stream);
// table of document starts of a whitespace-separated stream; scratch: doc_table_scratch_words(n) uint32 words.
// first_starts: whether structural 0 starts a document (true for a whole stream; for a shard, as the stream fold said)
size_t doc_table_scratch_words(uint32_t n);
cudaError_t launch_doc_table(const uint8_t *buf, const uint32_t *idx, uint32_t n, bool first_starts, uint32_t *scratch, sjb200_doc_boundary_t *table,
                             uint32_t capacity, uint32_t *ndocs_dev, cudaStream_t stream);
// sharded streaming passes: the shard's summary into every rank's window (x; layout in sjb200_params.h)
// (at: the word of this rank's block in every window)
cudaError_t launch_stream_summary(const uint8_t *buf, const uint32_t *idx, uint32_t count, uint32_t kept, uint32_t len, int walk, const Xchg &x,
                                  size_t at, cudaStream_t stream);
// ... and the rewrite of the (at most two) words of the final fix-up this rank holds
cudaError_t launch_store_words(uint32_t *idx, uint32_t nw, uint32_t p0, uint32_t v0, uint32_t p1, uint32_t v1, cudaStream_t stream);

// sharded RS / comma-delimited passes (modes 3..6), one shard of n structurals (less the stream's last one when the stream
// ends inside a string and this shard holds it); the rounds' words go to `at` + kDelim*At (sjb200_params.h).
// scratch: delim_scratch_words(n) words, kept from the carry round to the tail round
size_t delim_scratch_words(uint32_t n);
// carry round
cudaError_t launch_delim_carry(const uint8_t *buf, const uint32_t *idx, uint32_t n, uint32_t len, bool comma, uint32_t *scratch, const Xchg &x,
                               size_t at, cudaStream_t stream);
// filter round: the filter with the carried-in depth / run into the scratch (idx untouched); {filtered, separators, last
// separator, filtered before it} -> totals_host (pinned, valid once the stream is synchronised)
cudaError_t launch_delim_filter(const uint8_t *buf, uint32_t len, const uint32_t *idx, uint32_t n, bool comma, int depth_in, bool run_in, uint32_t *scratch,
                                uint32_t *totals_host, cudaStream_t stream);
const uint32_t *delim_filtered(const uint32_t *scratch);  // the filtered entries, shard-relative
cudaError_t launch_delim_publish_totals(uint32_t *scratch, uint32_t n, const Xchg &x, size_t at, cudaStream_t stream);
// tail round: the words this rank holds (src 1: filtered entry pos, 2: raw scanned word pos, 0: none; + add), published when
// `publish`; then the filtered entries go back to idx[0, filtered)
struct DelimTail {
  int32_t src[3];
  uint32_t pos[3];
  uint32_t add;
};
cudaError_t launch_delim_tail(uint32_t *scratch, uint32_t n, uint32_t *idx, const DelimTail &t, bool publish, const Xchg &x, size_t at,
                              cudaStream_t stream);

}  // namespace sjb200
