/*
 * sjb200.h -- C ABI of the H100 (sm_90a) stage-1 / minify / validate_utf8 library.
 *
 * This is the drop-in boundary for ONE hot path of simdjson (SURVEY.md section 8): it exports exactly
 * what a `simdjson::implementation` / `internal::dom_parser_implementation` back-end has to provide
 * for stage 1, minify and validate_utf8.  Plain pointers and sizes only; no C++ / torch types.
 * Every function returns a simdjson::error_code value as int (include/simdjson/error.h L19-54) and
 * never throws, prints or aborts (the reference's virtuals are all noexcept,
 * include/simdjson/implementation.h L97-128, internal/dom_parser_implementation.h L64-165).
 *
 * There is NO CPU fallback: if the CUDA runtime, the device (compute capability 10.x) or the kernel
 * image is unavailable, sjb200_create fails with SJB200_UNSUPPORTED_ARCHITECTURE, like
 * `unsupported_implementation` does (src/implementation.cpp L245-268).
 *
 * Reference interface each entry point replaces (paths relative to the simdjson tree):
 *   sjb200_create / _destroy / _set_capacity
 *        implementation::create_dom_parser_implementation   include/simdjson/implementation.h L97-101
 *        dom_parser_implementation::set_capacity             include/simdjson/generic/dom_parser_implementation.h L66-82
 *   sjb200_stage1
 *        dom_parser_implementation::stage1(buf,len,mode)     include/simdjson/internal/dom_parser_implementation.h L80
 *        (= json_structural_indexer::index<128>              src/generic/stage1/json_structural_indexer.h L193-397)
 *   sjb200_minify
 *        implementation::minify(buf,len,dst,dst_len)         include/simdjson/implementation.h L116
 *   sjb200_validate_utf8
 *        implementation::validate_utf8(buf,len)              include/simdjson/implementation.h L128
 * The *_dev variants take device pointers (input already resident in HBM); they are what the
 * roofline metric times.  The sharded variant is the per-GPU piece of a multi-GPU scan (section 8e).
 */
#ifndef SJB200_H
#define SJB200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define SJB200_API __attribute__((visibility("default")))
#else
#define SJB200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* simdjson::error_code values used by this path */
enum {
  SJB200_SUCCESS = 0,
  SJB200_CAPACITY = 1,
  SJB200_MEMALLOC = 2,
  SJB200_UTF8_ERROR = 11,
  SJB200_EMPTY = 13,
  SJB200_UNESCAPED_CHARS = 14,
  SJB200_UNCLOSED_STRING = 15,
  SJB200_UNSUPPORTED_ARCHITECTURE = 16,
  SJB200_UNEXPECTED_ERROR = 24
};

/* simdjson::stage1_mode (include/simdjson/internal/dom_parser_implementation.h L22-27) */
enum {
  SJB200_REGULAR = 0,
  SJB200_STREAMING_PARTIAL = 1,
  SJB200_STREAMING_FINAL = 2,
  SJB200_JSON_SEQUENCE_PARTIAL = 3,
  SJB200_JSON_SEQUENCE_FINAL = 4,
  SJB200_COMMA_DELIMITED_PARTIAL = 5,
  SJB200_COMMA_DELIMITED_FINAL = 6
};

typedef struct sjb200_ctx sjb200_ctx;

/* ---- lifetime: one context per dom_parser_implementation instance (own stream + scratch; contexts
 * are independent, so two parsers may run from two host threads concurrently, as document_stream's
 * stage-1 worker requires: include/simdjson/dom/document_stream-inl.h L16-85).
 * A context is used by ONE host thread and on ONE stream at a time: its look-back descriptors, ticket and flag words
 * are shared by all of its launches, which are therefore meant to run one after the other (calls that take a `stream`
 * may be given any stream, but consecutive calls on different streams must be ordered by the caller). */
SJB200_API int sjb200_create(int device, size_t capacity_bytes, sjb200_ctx **out);
SJB200_API void sjb200_destroy(sjb200_ctx *ctx);
SJB200_API int sjb200_set_capacity(sjb200_ctx *ctx, size_t capacity_bytes); /* > 0xFFFFFFFF -> CAPACITY */
SJB200_API size_t sjb200_capacity(const sjb200_ctx *ctx);
/* number of uint32 words of an index buffer for `capacity`: ROUNDUP(capacity,64)+9 */
SJB200_API size_t sjb200_index_words(size_t capacity_bytes);
SJB200_API int sjb200_device(const sjb200_ctx *ctx);
/* last CUDA error string seen by this context ("" if none); for diagnostics only */
SJB200_API const char *sjb200_last_cuda_error(const sjb200_ctx *ctx);
/* tuning knobs, mostly for tests and bench: "use_tma" (0/1), "grid" (CTAs, 0 = auto), "chunk_bytes", "copy_threads",
 * "ew_min_bytes" (stage-1 launches of at least this size use the emit-warp build of the kernel; 0 = never),
 * "time_kernel" (0/1: record CUDA events around the scan kernel on its launch stream); none changes results */
SJB200_API int sjb200_set_option(sjb200_ctx *ctx, const char *key, long value);
/* "kernel_ms" (last scan kernel, needs time_kernel=1), "launches" (kernels launched by this context so far),
 * "ew_launches" (of which on the emit-warp build),
 * "grid_index", "sm_count"; negative when unavailable */
SJB200_API double sjb200_get_stat(sjb200_ctx *ctx, const char *key);

/* tuning aid (option "debug_timeline"=1): per-tile phase timestamps of the last launch, 8 x uint64 per tile */
SJB200_API long sjb200_get_debug_timeline(sjb200_ctx *ctx, unsigned long long *out, size_t max_tiles);

/* page-lock / unlock caller-owned host memory (e.g. the parser's `new uint32_t[]` index array, whose deleter the
 * reference fixes: internal/dom_parser_implementation.h L175) so copies to it run at full PCIe speed; best effort */
SJB200_API int sjb200_pin_host_memory(sjb200_ctx *ctx, void *ptr, size_t bytes);
SJB200_API int sjb200_unpin_host_memory(sjb200_ctx *ctx, void *ptr);

/* ---- host-pointer entry points (copy in, scan, copy out).
 * idx_out: at least sjb200_index_words(capacity) words; on success and on UTF8_ERROR / EMPTY(after scan)
 * it holds n indexes followed by the reference's three sentinel words.  *n_inout is the parser's
 * n_structural_indexes: untouched on the early-return paths exactly like the reference
 * (CAPACITY, len==0, UNCLOSED_STRING, UNESCAPED_CHARS). */
SJB200_API int sjb200_stage1(sjb200_ctx *ctx, const uint8_t *buf, size_t len, int mode, uint32_t *idx_out, uint32_t *n_inout);
/* dst needs len bytes (the reference's tests give it exactly len: tests/dom/basictests.cpp L1916). */
SJB200_API int sjb200_minify(sjb200_ctx *ctx, const uint8_t *buf, size_t len, uint8_t *dst, size_t *dst_len);
/* returns 1 valid / 0 invalid; a CUDA failure reports 0 and sets sjb200_last_cuda_error.  No size limit (inputs beyond
 * 4 GiB are validated piece by piece); sjb200_minify and the *_dev variants accept at most 0xFFFFFFFF bytes per call
 * (CAPACITY beyond that -- a deviation from the reference, whose minify is unbounded; see INTEGRATION.md). */
SJB200_API int sjb200_validate_utf8(sjb200_ctx *ctx, const uint8_t *buf, size_t len);

/* ---- device-resident entry points.  d_* are device pointers on the context's device; `stream` is a
 * cudaStream_t (NULL = the context's own stream).  The calls return after the result is known
 * (they synchronise the stream once).  d_idx needs sjb200_index_words(len) words. */
SJB200_API int sjb200_stage1_dev(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, uint32_t *n_inout,
                      void *stream);
SJB200_API int sjb200_minify_dev(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, uint8_t *d_dst, size_t *dst_len, void *stream);
SJB200_API int sjb200_validate_utf8_dev(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, void *stream);

/* many documents per call: all scans are queued back to back, one host wait, then each document's finish().
 * (what a caller with a corpus / NDJSON rows resident in HBM uses instead of a loop of sjb200_stage1_dev) */
typedef struct {
  const uint8_t *d_buf;          /* in: device pointer */
  size_t len;                    /* in */
  uint32_t *d_idx;               /* in: device index buffer, sjb200_index_words(len) words */
  uint32_t n_structural_indexes; /* in/out, like sjb200_stage1_dev's n_inout */
  int error;                     /* out: simdjson::error_code */
} sjb200_doc;
SJB200_API int sjb200_stage1_dev_batch(sjb200_ctx *ctx, sjb200_doc *docs, int ndocs, int mode, void *stream);

/* every place a document of a whitespace-separated stream (NDJSON, concatenated documents) starts, from the
 * device-resident output (d_idx, n) of a stage-1 call: (structural index, byte offset) pairs in stream order, built on
 * the device (SURVEY.md 8(f) row 1).  Structural i >= 1 starts a document when it is a value or an opening bracket and
 * structural i-1 is neither an opening bracket nor ',' / ':' -- the predicate of find_next_document_index
 * (src/generic/stage1/find_next_document_index.h L60-88), applied to every position instead of the last one only, so a
 * consumer can hand the documents of ONE big stage-1 pass to many stage-2 workers instead of discovering them window by
 * window (include/simdjson/dom/document_stream-inl.h L245-271).  *ndocs_out = number of starts found (entries beyond
 * `capacity` are not stored). */
typedef struct {
  uint32_t index; /* structural index at which a document starts */
  uint32_t byte;  /* = structural_indexes[index] */
} sjb200_doc_boundary;
SJB200_API int sjb200_document_table_dev(sjb200_ctx *ctx, const uint8_t *d_buf, const uint32_t *d_idx, uint32_t n, sjb200_doc_boundary *d_table,
                              uint32_t capacity, uint32_t *ndocs_out, void *stream);

/* stage-2-lite on the device (SURVEY.md 8(f) row 4): from the device-resident output (d_idx, n) of a stage-1 call, what
 * the reference's stage 2 decides about every token from its bytes alone -- the leaves of json_iterator::visit_primitive
 * (src/generic/stage2/json_iterator.h L338-360) -- for all tokens at once:
 *   d_type[k]     the tape_type char of structural k (include/simdjson/internal/tape_type.h L10-24): '{' '}' '[' ']'
 *                 '"' 'l' (int64) 'u' (uint64) 'd' (float) 't' 'f' 'n'; ':' and ',' for those operators (they have no
 *                 tape entry); 0 for a token in error
 *   d_payload[k]  '"': offset of the string's record in d_strbuf (the tape payload of a string); 'l' / 'u': the value
 *                 (numberparsing::parse_number, include/simdjson/generic/numberparsing.h L860-961); 'd': byte offset one
 *                 past the number (floats are validated by grammar and delimited, not converted -- the reference also
 *                 rejects floats whose value is infinite, L765-813); 0 type: the error_code (STRING_ERROR 5, T/F/N_ATOM
 *                 _ERROR 6/7/8, NUMBER_ERROR 9, BIGINT_ERROR 10, TAPE_ERROR 3); other types: 0
 *   d_strbuf      the document's string buffer, byte-identical to dom::document::string_buf after dom::parser::parse of
 *                 the same document: per string, in document order, [uint32 length][unescaped bytes][0]
 *                 (tape_builder::visit_string, src/generic/stage2/tape_builder.h L186-205; stringparsing::parse_string,
 *                 stringparsing.h L146-190 -- the batched form of the dom_parser_implementation::parse_string virtual,
 *                 include/simdjson/internal/dom_parser_implementation.h L124).  sjb200_string_buf_capacity(len) bytes
 *                 always suffice (the reference's own sizing, include/simdjson/dom/document-inl.h L54).
 * Scalars are judged as values inside an array or object (visit_primitive, not visit_root_primitive).  Not done here:
 * the nesting grammar (the sequential part of stage 2).  Returns out->error: the error of the first token in error in
 * document order (what a sequential stage 2 would have stopped at, token-level errors only), CAPACITY when d_strbuf is
 * too small (nothing is written to it then; out->string_bytes says how much is needed), else SUCCESS. */
typedef struct {
  int error;
  uint32_t first_error_index; /* structural index of the first token in error, 0xFFFFFFFF when none */
  uint32_t n_strings;
  uint64_t string_bytes;      /* bytes of d_strbuf in use */
} sjb200_tokens_result;
SJB200_API size_t sjb200_string_buf_capacity(size_t len);
SJB200_API int sjb200_tokens_dev(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, const uint32_t *d_idx, uint32_t n, uint8_t *d_type, uint64_t *d_payload,
                      uint8_t *d_strbuf, size_t strbuf_capacity, sjb200_tokens_result *out, void *stream);

/* split form of the same calls for pipelining / timing: enqueue returns as soon as the work is on the
 * stream, finish waits for it and completes the reference's finish() logic. */
SJB200_API int sjb200_stage1_dev_enqueue(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, void *stream);
SJB200_API int sjb200_stage1_dev_finish(sjb200_ctx *ctx, uint32_t *n_inout);
SJB200_API int sjb200_minify_dev_enqueue(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, uint8_t *d_dst, void *stream);
SJB200_API int sjb200_minify_dev_finish(sjb200_ctx *ctx, size_t *dst_len);
SJB200_API int sjb200_validate_utf8_dev_enqueue(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, void *stream);
SJB200_API int sjb200_validate_utf8_dev_finish(sjb200_ctx *ctx);

/* ---- multi-GPU: one shard of a document per GPU (SURVEY.md section 8e).
 * A shard is scanned with a given incoming scanner state (bit0 escape, bit1 in-string, bit2
 * previous-byte-was-scalar); the call reports the shard's 6-bit carry transducer, which is
 * independent of the incoming state, so ranks can all-gather {ttable,count} once, fold their true
 * incoming state, and re-scan only if their speculation (state 0) was wrong.
 * Shards must be cut where the next byte is not a UTF-8 continuation byte (sjb200_shard_cut). */
typedef struct {
  uint32_t ttable;     /* T(e): bit0 esc(0) bit1 parity(0) bit2 scalar(0) bit3 esc(1) bit4 parity(1) bit5 scalar(1) */
  uint32_t state_out;  /* ttable applied to state_in */
  uint32_t flags;      /* bit0 utf-8 error, bit1 unescaped control char in string, bit2 internal error */
  uint32_t reserved;
  uint64_t count;      /* structurals found in this shard (indexes are shard-relative) */
} sjb200_shard_result;
SJB200_API int sjb200_stage1_shard_dev(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, uint32_t state_in, int last_shard,
                            uint32_t *d_idx, sjb200_shard_result *out, void *stream);
/* the speculative pass (incoming state 0) without host synchronisation: d_result is DEVICE memory, 24 bytes
 * {uint64 count; uint32 state_out; uint32 ttable; uint32 flags; uint32 reserved}, e.g. the send buffer of an
 * all-gather enqueued behind the scan on the same stream */
SJB200_API int sjb200_stage1_shard_dev_enqueue(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, uint32_t *d_idx, void *d_result,
                                    void *stream);
/* ---- the sharded scan as one call per rank, exchange fused into the scan kernel (no collective launch).
 * One sjb200_comm per rank (one process per GPU, or several contexts in one process).  Each comm owns an exchange
 * window in its device's memory; peers map each other's windows (CUDA IPC across processes: get_handle -> exchange the
 * 64-byte handles by any means, e.g. one NCCL/gloo all-gather at start-up -> connect).  During a pass the scan
 * kernel's last CTA stores the shard's 16-byte record {count, state, transducer, flags} straight into every rank's
 * window over NVLink; finish() folds the true incoming state / 64-bit index base from the local window and, only if
 * some rank's speculation (state 0) was wrong, re-scans that rank and runs a second round.  Indexes stay
 * shard-relative (uint32) + base, like document_stream's batch_start + structural_indexes[i]
 * (include/simdjson/dom/document_stream-inl.h L250).  Up to 32 passes may be in flight per rank. */
typedef struct sjb200_comm sjb200_comm;
#define SJB200_COMM_HANDLE_BYTES 64
typedef struct {
  uint64_t count;        /* structurals of this shard (after a re-scan: the corrected count) */
  uint64_t base;         /* structurals of all earlier shards: global index i of this shard = base + i */
  uint64_t total_count;  /* structurals of all shards */
  uint32_t state_in;     /* true scanner state entering this shard (0 = the speculation held) */
  uint32_t state_out;
  uint32_t final_state;  /* state after the last shard (bit1: the document ends inside a string) */
  uint32_t flags;        /* this shard: bit0 utf-8 error, bit1 unescaped control char in string, bit2 internal */
  uint32_t flags_all;    /* union over all shards */
  uint32_t rescanned;    /* 1: this rank scanned twice */
} sjb200_sharded_result;
SJB200_API int sjb200_comm_create(sjb200_ctx *ctx, int rank, int nranks /* <= 8 */, sjb200_comm **out);
SJB200_API void sjb200_comm_destroy(sjb200_comm *comm);
SJB200_API int sjb200_comm_get_handle(sjb200_comm *comm, void *handle /* SJB200_COMM_HANDLE_BYTES */);
SJB200_API int sjb200_comm_connect(sjb200_comm *comm, const void *handles /* nranks x 64 bytes, by rank */);
SJB200_API int sjb200_comm_connect_local(sjb200_comm *comm, sjb200_comm *const *all /* nranks comms of this process, by rank */);
SJB200_API int sjb200_stage1_sharded(sjb200_comm *comm, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx,
                          sjb200_sharded_result *out, void *stream);
SJB200_API int sjb200_stage1_sharded_enqueue(sjb200_comm *comm, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx,
                                  void *stream);
SJB200_API int sjb200_stage1_sharded_finish(sjb200_comm *comm, sjb200_sharded_result *out); /* completes the oldest pass in flight */

/* fold: state entering shard r given the ttables of shards 0..r-1 and the document's initial state 0 */
SJB200_API uint32_t sjb200_fold_state(const uint32_t *ttables, int nshards_before);
/* largest cut <= nominal such that buf[cut] is not a UTF-8 continuation byte (host pointer) */
SJB200_API size_t sjb200_shard_cut(const uint8_t *buf, size_t len, size_t nominal);
/* the same, preferring the byte after a raw line feed within `window` bytes below nominal: a raw 0x0A cannot occur
 * inside a JSON string, so for valid input the next shard starts in state 0 and the speculation always holds */
SJB200_API size_t sjb200_shard_cut_line(const uint8_t *buf, size_t len, size_t nominal, size_t window);

#ifdef __cplusplus
}
#endif
#endif /* SJB200_H */
