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
 * roofline metric times.  The sharded variants (stage 1, minify, validate_utf8, stage-2-lite) are the per-GPU pieces of a multi-GPU
 * pass over one buffer cut by byte range (section 8e).
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
  SJB200_INCORRECT_TYPE = 17,
  SJB200_NUMBER_OUT_OF_RANGE = 18,
  SJB200_INDEX_OUT_OF_BOUNDS = 19,
  SJB200_NO_SUCH_FIELD = 20,
  SJB200_INVALID_JSON_POINTER = 22,
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
 * "time_kernel" (0/1: record CUDA events around the scan kernel on its launch stream), "pdl" (0/1, default 1: the
 * scan launches of one sjb200_stage1_dev_batch call after the first may start while the previous one still runs),
 * "launch_stamps" (0/1: sjb200_get_launch_stamps); none changes results */
SJB200_API int sjb200_set_option(sjb200_ctx *ctx, const char *key, long value);
/* "kernel_ms" (last scan kernel, needs time_kernel=1), "kernel_ms_mean" (the scan kernels since the previous query),
 * both per document: a launch that scans several documents (sjb200_stage1_dev_batch) counts its duration divided by
 * their number, and a sjb200_stage1_dev_batch call counts the span from its first scan launch to the end of its last
 * one (launches may overlap), divided by its documents; "launches" (kernels launched by this context so far),
 * "grid_index", "sm_count"; negative when unavailable */
SJB200_API double sjb200_get_stat(sjb200_ctx *ctx, const char *key);

/* tuning aid (option "debug_timeline"=1): per-tile phase timestamps of the last launch, 8 x uint64 per tile */
SJB200_API long sjb200_get_debug_timeline(sjb200_ctx *ctx, unsigned long long *out, size_t max_tiles);
/* tuning aid (option "launch_stamps"=1): for every scan launch of the last sjb200_stage1_dev_batch call, the globaltimer
 * (ns) at its first CTA's entry and at its last CTA's exit (0 for a group of one document); returns the launches copied */
SJB200_API long sjb200_get_launch_stamps(sjb200_ctx *ctx, unsigned long long *out, size_t max_launches);

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

/* many documents per call: consecutive documents share one scan launch (up to 64 per launch), the launches are queued
 * back to back, one host wait, then each document's finish().  A launch ends before a document whose input or index
 * buffer overlaps the index buffer of an earlier document of the launch, or whose index buffer overlaps such a
 * document's input, so results are those of a loop of sjb200_stage1_dev in order.
 * (what a caller with a corpus / NDJSON rows resident in HBM uses instead of that loop) */
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

/* JSON Pointer lookup on the device for every document of a stream: dom::element::at_pointer
 * (include/simdjson/dom/element-inl.h L410-446, object-inl.h L104-147, array-inl.h L94-121, jsonpathutil.h L20-50) of
 * every pointer in every document, batched, over the output of sjb200_tokens_dev (d_type, d_payload for n structurals,
 * and its string buffer d_strbuf, of which string_bytes are in use).  d_docs / ndocs: a table from
 * sjb200_document_table_dev; NULL or 0 = one document, structurals [0, n).  Document d is structurals
 * [d_docs[d].index, d_docs[d + 1].index) (the last one: up to n).  pointers / pointer_lens: host strings (not
 * NUL-terminated).  d_out: device memory, npointers x ndocs results (1 per pointer without a table), pointer-major:
 * d_out[p * ndocs + d].  The results stay on the device; the call synchronises its stream once before it returns.
 *
 * A result is {SUCCESS, structural index of the selected value} -- d_type / d_payload / d_idx at that index give its
 * type, its value or string-record offset, and its byte offset (a 'd' value is the span of its number, as for
 * sjb200_tokens_dev) -- or {error, 0xFFFFFFFF} with the error at_pointer returns: INCORRECT_TYPE, INDEX_OUT_OF_BOUNDS,
 * NO_SUCH_FIELD or INVALID_JSON_POINTER, in the reference's order of decision.  Two errors come first:
 *   - a table entry that is not above the one before it, or not below n: UNEXPECTED_ERROR for that document;
 *   - a token in error (d_type 0) in the document: {its d_payload error code, its structural index}, for the first such
 *     token -- what dom::parser::parse reports for a document whose grammar is otherwise valid.
 * Deviations from the reference: documents that parse rejects for their nesting get an error or an index inside the
 * document, never a fault (sjb200_document_errors_dev gives the exact parse error: drop the results of the documents
 * whose verdict there is not SUCCESS); max_depth is not enforced; root scalars are judged as sjb200_tokens_dev judges them; the walk
 * follows the DOM API, not On-Demand.  A walk never reads outside [0, n) of the token arrays or [0, string_bytes) of the
 * string buffer.
 * Returns SUCCESS; CAPACITY, before any launch, beyond one of the limits below; MEMALLOC or UNEXPECTED_ERROR for a CUDA
 * failure or bad arguments. */
#define SJB200_POINTER_MAX_POINTERS 65536   /* pointers per call */
#define SJB200_POINTER_MAX_TOKENS 1024      /* reference tokens per pointer */
#define SJB200_POINTER_MAX_BYTES 1048576    /* bytes of all pointers of a call */
typedef struct {
  int32_t error;
  uint32_t index;
} sjb200_pointer_result;
SJB200_API int sjb200_at_pointer_dev(sjb200_ctx *ctx, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                     size_t string_bytes, const sjb200_doc_boundary *d_docs, uint32_t ndocs, const char *const *pointers,
                                     const size_t *pointer_lens, int npointers, sjb200_pointer_result *d_out, void *stream);

/* Typed columns from JSON Pointer results on the device: for every row of d_rows (nrows results of sjb200_at_pointer_dev,
 * as they are: one pointer's column is d_rows + p * ndocs, and several pointers go in one call), what one DOM getter
 * returns on the element the row selects.  (d_type, d_payload, n, d_strbuf, string_bytes) is the output of
 * sjb200_tokens_dev the lookup ran on.  Row r, decided in this order:
 *   1. a row in error stays in error: d_err[r] = its error, d_row_type[r] = 0, the value 0, the string empty;
 *   2. an index >= n, or at a token that is not a value (',' ':' '}' ']' or 0), is UNEXPECTED_ERROR with d_row_type 0;
 *      so is (STRING only, where the record is read) a string whose record [u32 length][bytes][0] does not lie inside
 *      [0, string_bytes).  Nothing outside [0, n) of the token arrays or [0, string_bytes) of d_strbuf is read;
 *   3. d_row_type[r] = the tape type char of the value ('{' '[' '"' 'l' 'u' 'd' 't' 'f' 'n'), and d_err[r] / the value
 *      are the getter's (include/simdjson/dom/element-inl.h):
 *      INT64        get_int64: 'l' its value; 'u' its value up to INT64_MAX, else NUMBER_OUT_OF_RANGE
 *      UINT64       get_uint64: 'u' its value; 'l' its value when >= 0, else NUMBER_OUT_OF_RANGE
 *      BOOL         get_bool: 't' 1, 'f' 0
 *      STRING       get_string: the exact bytes of the record ("\u0000" kept, no terminator), Arrow large_string layout:
 *                   d_offsets[0] = 0, row r is d_bytes[d_offsets[r], d_offsets[r + 1]), a row in error has length 0
 *      ARRAY_SIZE   get_array().size(): the elements of a '[' (the structurals at its depth other than ',')
 *      OBJECT_SIZE  get_object().size(): the fields of a '{' (its strings followed by ':'; duplicate keys count)
 *      Sizes saturate at 0xFFFFFF like the tape's scope count (src/generic/stage2/tape_builder.h, cntsat).  Any other
 *      type is INCORRECT_TYPE; a 'd' value (a float, not converted here: see sjb200_column_double_dev) is INCORRECT_TYPE under INT64 / UINT64
 *      as in the reference, and its row type tells it apart.  On an error the value is 0.
 * d_values: nrows uint64 (INT64: the int64 bits; UINT64; the sizes) or nrows uint8 (BOOL); not used for STRING.  d_offsets
 * (nrows + 1 int64) and d_bytes (bytes_capacity bytes) are used by STRING only.  Outputs are device memory and stay there;
 * nothing outside the rows and no byte of d_bytes past out->string_bytes is written.  The call synchronises its stream
 * once.  Its device scratch (kept by the context) is about 30 bytes per row, plus for STRING bytes_capacity / 512.  nrows = 0 writes d_offsets[0] = 0 (STRING) and nothing else.
 * Deviations: the rows carry no document end, so a size walk stops at n -- a container the reference rejects for its
 * nesting is counted up to there, never a fault (as for sjb200_at_pointer_dev); 1e400 and other infinite floats are 'd'
 * rows here where the reference fails the parse.
 * Returns SUCCESS; CAPACITY for STRING when bytes_capacity is less than the column's bytes (d_err, d_row_type and
 * d_offsets are written, nothing to d_bytes, out->string_bytes holds the need -- the contract of sjb200_tokens_dev's
 * d_strbuf); UNEXPECTED_ERROR for an unknown kind or a NULL output the kind needs; MEMALLOC or UNEXPECTED_ERROR for a
 * CUDA failure. */
enum {
  SJB200_COLUMN_INT64 = 1,        /* element::get_int64            -> int64_t  values */
  SJB200_COLUMN_UINT64 = 2,       /* element::get_uint64           -> uint64_t values */
  SJB200_COLUMN_BOOL = 3,         /* element::get_bool             -> uint8_t  values (0 / 1) */
  SJB200_COLUMN_STRING = 4,       /* element::get_string           -> int64 offsets[nrows + 1] + bytes */
  SJB200_COLUMN_ARRAY_SIZE = 5,   /* element::get_array().size()   -> uint64_t values */
  SJB200_COLUMN_OBJECT_SIZE = 6   /* element::get_object().size()  -> uint64_t values */
};
typedef struct {
  uint32_t rows_in_error;
  uint32_t reserved;
  uint64_t string_bytes;          /* STRING: bytes of the packed column (under CAPACITY: the bytes needed) */
} sjb200_column_result;
SJB200_API int sjb200_column_dev(sjb200_ctx *ctx, int kind, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                 size_t string_bytes, const sjb200_pointer_result *d_rows, uint32_t nrows, int32_t *d_err, uint8_t *d_row_type,
                                 void *d_values, int64_t *d_offsets, uint8_t *d_bytes, size_t bytes_capacity, sjb200_column_result *out,
                                 void *stream);

/* Float columns from JSON Pointer results on the device: for every row of d_rows (as for sjb200_column_dev), what
 * element::get_double returns on the element the row selects, correctly rounded.  (d_buf, len, d_idx) are the input and
 * the structurals of the stage-1 call, (d_type, d_payload, n) the output of sjb200_tokens_dev on them; a 'd' token k is
 * the number d_buf[d_idx[k], d_payload[k]).  Row r, decided in this order:
 *   1. a row in error stays in error: d_err[r] = its error, d_row_type[r] = 0, d_values[r] = +0.0;
 *   2. an index >= n, at a token that is not a value, or at a 'd' token whose span is empty, not inside [0, len) or not
 *      a JSON number, is UNEXPECTED_ERROR with d_row_type 0.  Nothing outside [0, n) of the token arrays or [0, len) of
 *      d_buf is read;
 *   3. d_row_type[r] = the tape type char of the value, and
 *      'd'       the binary64 nearest to the number's text (ties to even), as the reference's parse_number writes it;
 *                NUMBER_ERROR with the value 0 when that is infinite
 *      'l' 'u'   double(int64) / double(uint64), rounded to nearest even ("-0" is an 'l' 0 and gives +0.0; "-0.0" gives
 *                -0.0)
 *      others    INCORRECT_TYPE, the value 0.
 * Deviation: an infinite float ("1e400") fails the reference's whole parse; here only its row is NUMBER_ERROR (the tokens
 * already accept it, see sjb200_tokens_dev).  out->rows_in_error counts the rows in error; out->string_bytes is 0.  The
 * call synchronises its stream once; nothing outside the rows of the outputs is written, and nrows = 0 writes nothing.  A
 * number of more than 64 bytes is read by a CTA, and one whose value the Eisel-Lemire step leaves open is decided
 * exactly on its first 768 significant digits (the rest only break ties).  Device scratch (kept by the context): 8
 * bytes per row.  Returns SUCCESS; UNEXPECTED_ERROR for a NULL output or input that is needed; MEMALLOC or
 * UNEXPECTED_ERROR for a CUDA failure. */
SJB200_API int sjb200_column_double_dev(sjb200_ctx *ctx, const uint8_t *d_buf, size_t len, const uint32_t *d_idx, const uint8_t *d_type,
                                        const uint64_t *d_payload, uint32_t n, const sjb200_pointer_result *d_rows, uint32_t nrows, int32_t *d_err,
                                        uint8_t *d_row_type, double *d_values, sjb200_column_result *out, void *stream);

/* Stage-2 grammar on the device: for every document, the error json_iterator::walk_document
 * (src/generic/stage2/json_iterator.h L120-244, with tape_builder) returns, from the output of sjb200_tokens_dev (d_type,
 * d_payload for n structurals of a regular-mode stage 1 that succeeded).  No table (d_docs NULL or ndocs 0): one document
 * [0, n), as dom::parser::parse judges it (n = 0: {EMPTY, 0}).  With a table from sjb200_document_table_dev: document d
 * is [d_docs[d].index, d_docs[d + 1].index) (the last one: up to n), as stage2_next from its first structural judges it
 * (document_stream-inl.h L250-269); a walk that ends before the document's end is a TAPE_ERROR at the first structural
 * left over, one that would read the structural at the end a TAPE_ERROR at the end.
 * d_out (device memory, one per document): {error, structural index at which it was decided}, or {SUCCESS, one past the
 * document's value}.  *out: the documents in error and the first of them.  One stream synchronise.  A caller of
 * sjb200_at_pointer_dev gets the exact parse error by dropping the results of documents whose verdict is not SUCCESS.
 * Deviations: an infinite float (1e400) is SUCCESS (the tokens check only float grammar); a root token starting with a
 * byte below '0' other than '-' (+1, #) is NUMBER_ERROR, not TAPE_ERROR (the tokens do not keep the byte); the last
 * document of a stream that wants a value past n is a TAPE_ERROR at n (the reference judges its padding byte there).
 * Returns SUCCESS; CAPACITY, before any launch and with nothing written, for max_depth 0 or above
 * SJB200_DOCUMENT_MAX_DEPTH; UNEXPECTED_ERROR when the table is not strictly ascending or has an entry at or above n
 * (every result {UNEXPECTED_ERROR, 0xFFFFFFFF}); MEMALLOC or UNEXPECTED_ERROR for a CUDA failure or bad arguments. */
#define SJB200_DOCUMENT_MAX_DEPTH 4096
typedef struct {
  int32_t error;   /* simdjson::error_code */
  uint32_t index;  /* structural index at which it was decided; SUCCESS: one past the document's value */
} sjb200_document_error;
typedef struct {
  uint32_t ndocs_in_error;
  uint32_t first_doc_in_error;  /* 0xFFFFFFFF when none: where parse_many stops */
} sjb200_document_errors_result;
SJB200_API int sjb200_document_errors_dev(sjb200_ctx *ctx, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n,
                                          const sjb200_doc_boundary *d_docs, uint32_t ndocs, size_t max_depth,
                                          sjb200_document_error *d_out, sjb200_document_errors_result *out, void *stream);

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
 * kernel's last CTA stores the shard's 16-byte record {count, state, transducer, flags, kind} straight into every rank's
 * window over NVLink; finish() folds the true incoming state / 64-bit index base from the local window and, only if
 * some rank's speculation (state 0) was wrong, re-scans that rank and runs a second round.  Indexes stay
 * shard-relative (uint32) + base, like document_stream's batch_start + structural_indexes[i]
 * (include/simdjson/dom/document_stream-inl.h L250).  Up to 32 passes may be in flight per rank. */
typedef struct sjb200_comm sjb200_comm;
#define SJB200_COMM_HANDLE_BYTES 64
typedef struct {        /* counts are structurals (stage 1), kept bytes (minify) or 0 (validate_utf8) */
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

/* minify and validate_utf8 sharded the same way, on the same comm and window.  A pass is stage 1, minify or
 * validate_utf8 (its kind, carried in the record); passes of all kinds may be in flight together, up to the limit above,
 * when every rank enqueues the same sequence of kinds.  Each finish completes the oldest pass in flight, which must be
 * of its kind (else UNEXPECTED_ERROR and the pass stays in flight); a peer that published another kind for the same
 * pass makes finish fail with UNEXPECTED_ERROR (validate: -1) and sets sjb200_last_cuda_error.  len >= 1.
 *
 * minify: d_dst needs len bytes; this shard's kept bytes are d_dst[0, out->count).  out->base = their offset in the
 *   minified document, out->total_count = its length; state_in / final_state / flags / flags_all / rescanned as for stage
 *   1, except that minify validates nothing, so only the internal-error bit of the flags is ever set.  Cuts may be at any byte (minify does not look at UTF-8; escape and in-string cross the cut in the state).  Only
 *   bits 0-1 of the state change which bytes are kept, so a rank re-minifies only when (state_in & 3) != 0, and the second
 *   round runs only when that holds for some rank.  When final_state bit 1 is set (the document ends inside a string)
 *   every rank returns UNCLOSED_STRING, like sjb200_minify_dev, with `out` filled.  The outputs stay on their ranks:
 *   gathering them is one copy of d_dst[0, count) to [base, base + count) per rank, by the caller.
 * validate_utf8: finish returns 1 when every shard is valid UTF-8, 0 when one is not, negative on a CUDA failure or an
 *   exchange timeout.  Cuts must be at character boundaries (sjb200_shard_cut), as for stage 1: then every shard checks
 *   its own end and the AND of the shards' verdicts is the verdict on the whole buffer.  The records carry count 0,
 *   state 0 and transducer 0, so no second round ever runs. */
SJB200_API int sjb200_minify_sharded_enqueue(sjb200_comm *comm, const uint8_t *d_shard, size_t len, uint8_t *d_dst, void *stream);
SJB200_API int sjb200_minify_sharded_finish(sjb200_comm *comm, sjb200_sharded_result *out);
SJB200_API int sjb200_minify_sharded(sjb200_comm *comm, const uint8_t *d_shard, size_t len, uint8_t *d_dst, sjb200_sharded_result *out,
                          void *stream);
SJB200_API int sjb200_validate_utf8_sharded_enqueue(sjb200_comm *comm, const uint8_t *d_shard, size_t len, void *stream);
SJB200_API int sjb200_validate_utf8_sharded_finish(sjb200_comm *comm, sjb200_sharded_result *out);
SJB200_API int sjb200_validate_utf8_sharded(sjb200_comm *comm, const uint8_t *d_shard, size_t len, sjb200_sharded_result *out, void *stream);

/* stage 1 of a whitespace-separated stream (NDJSON, concatenated documents) sharded the same way, with the whole
 * stream's finish(): `mode` is SJB200_REGULAR, SJB200_STREAMING_PARTIAL or SJB200_STREAMING_FINAL (3-6, the RS and
 * comma-delimited streams, are rejected with UNEXPECTED_ERROR: they go through sjb200_stage1_sharded_delimited, whose
 * result describes a compacted array).  Every rank passes the same mode; last_shard = 1 on the last rank only.  In the streaming modes the
 * last shard alone is trimmed of a partial UTF-8 character at its end (a shard that trims to nothing still takes part).
 * Cuts at character boundaries (sjb200_shard_cut / sjb200_shard_cut_line).  A stream pass has its own kind, so a rank
 * whose peers enqueued another kind for the same pass fails with UNEXPECTED_ERROR.
 *
 * finish returns, on every rank, the error code stage1(whole buffer, mode) returns, and:
 *   n      that call's n_structural_indexes (0 on the paths where it leaves n untouched: UNCLOSED_STRING in regular
 *          mode, UNESCAPED_CHARS, a stream that trims to nothing, an internal error);
 *   kept   how many of this shard's structurals are among the first n: d_idx[0, kept) + bytes_before are global
 *          structurals [shard.base, shard.base + kept);
 *   d_idx  gathered as G = concat over ranks of d_idx[0, shard.count) + bytes_before, followed by the last rank's three
 *          words after its count (the first two + its bytes_before), G[0, n + 3) is the whole call's index array up to
 *          n + 3.  In streaming-final mode the words at m = n and m + 1 that the reference rewrites are rewritten by the
 *          ranks that hold them, shard-relative (modulo 2^32);
 *   total_bytes  the stream's length after the trim (word m of streaming-final mode);
 *   first_starts_document  whether this shard's structural 0 starts a document (the predicate of
 *          sjb200_document_table_dev, applied across the cut to the last structural of the previous shard that has one).
 * Streaming modes run one more host-synchronised round than sjb200_stage1_sharded: every rank stores a small summary of
 * its shard (walked back from its last structural to its last document start) into every window and folds them. */
typedef struct {
  sjb200_sharded_result shard;    /* the fold of the scan, as sjb200_stage1_sharded_finish reports it */
  uint64_t n;
  uint64_t kept;
  uint64_t bytes_before;          /* byte offset of this shard in the stream */
  uint64_t total_bytes;
  uint32_t first_starts_document;
  uint32_t reserved;
} sjb200_sharded_stream_result;
SJB200_API int sjb200_stage1_sharded_stream_enqueue(sjb200_comm *comm, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                         void *stream);
SJB200_API int sjb200_stage1_sharded_stream_finish(sjb200_comm *comm, sjb200_sharded_stream_result *out);
SJB200_API int sjb200_stage1_sharded_stream(sjb200_comm *comm, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                 sjb200_sharded_stream_result *out, void *stream);

/* stage 1 of an RS-delimited (RFC 7464, modes SJB200_JSON_SEQUENCE_*) or comma-delimited (SJB200_COMMA_DELIMITED_*)
 * stream sharded the same way, with the whole stream's filter and finish().  `mode` is 3..6 (0-2 are rejected with
 * UNEXPECTED_ERROR: use sjb200_stage1_sharded_stream).  Same rules as that call: every rank passes the same mode,
 * last_shard = 1 on the last rank only, cuts at character boundaries, only the last shard is trimmed of a partial UTF-8
 * character (a shard that trims to nothing still takes part).  A delimited pass has its own kind: a rank whose peers
 * enqueued another kind for the same pass fails with UNEXPECTED_ERROR.
 *
 * finish returns, on every rank, the error code stage1(whole buffer, mode) returns, and:
 *   stream.n      that call's n_structural_indexes (0 where it leaves n untouched);
 *   filtered      this shard's entries after the filter: d_idx[0, filtered), shard-relative, in stream order;
 *   filtered_before  the filtered entries of all earlier ranks (the global position of d_idx[0]);
 *   stream.kept   how many of them are among the first n (d_idx[0, kept) + bytes_before);
 *   stream.bytes_before, stream.total_bytes, stream.first_starts_document  as for sjb200_stage1_sharded_stream, over the
 *                 filtered array (so sjb200_document_table_shard_dev works unchanged on d_idx[0, kept));
 *   tail          the whole call's index words n, n+1, n+2 (absolute, uint32): the next batch start (partial modes) or
 *                 the stream's length (final modes), then what the reference's in-place filter leaves behind.
 * Gathered as G = concat over ranks of (d_idx[0, kept) + bytes_before) (mod 2^32), followed by tail[0..2], G[0, n + 3)
 * is the whole call's index array up to n + 3.  The words of d_idx past `filtered` are unspecified.
 * Three host-synchronised rounds follow the scan's: a carry round (bracket depth / separator run entering each shard), a
 * filter round (filter counts, last separator, the walks of find_next_document_index) and a tail round. */
typedef struct {
  sjb200_sharded_stream_result stream;  /* n, kept count entries of the FILTERED array */
  uint64_t filtered;
  uint64_t filtered_before;
  uint32_t tail[3];
  uint32_t reserved;
} sjb200_sharded_delimited_result;
SJB200_API int sjb200_stage1_sharded_delimited_enqueue(sjb200_comm *comm, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                            void *stream);
SJB200_API int sjb200_stage1_sharded_delimited_finish(sjb200_comm *comm, sjb200_sharded_delimited_result *out);
SJB200_API int sjb200_stage1_sharded_delimited(sjb200_comm *comm, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                    sjb200_sharded_delimited_result *out, void *stream);

/* stage-2-lite (sjb200_tokens_dev) sharded the same way, on the same comm and window: every rank runs the token kernels
 * on its shard, and the kernel that scans the string-buffer sums stores the shard's record and totals into every rank's
 * window.  (d_idx, n) is a structural list of this shard from a sharded stage-1 pass (sjb200_stage1_sharded: count;
 * stream and delimited passes: kept, over d_idx as that pass left it), state_in that pass's folded state_in, len the shard
 * length it used (the last rank of a streaming pass: after the trim).  len and n may be 0.  A tokens pass has its own kind.
 *
 * The cut before a shard must be clean: state_in == 0 (the byte before it is whitespace, an operator or a closing quote),
 * so that no token spans it.  Cuts after a raw line feed (sjb200_shard_cut_line) are clean for every input stage 1
 * accepts without UNESCAPED_CHARS.  A token that spans a cut is detected, not handled: finish returns UNEXPECTED_ERROR.
 *
 * Outputs stay on their ranks, shard-relative: d_type[0, n), d_payload[0, n) and d_strbuf[0, string_bytes).  Gathered as
 * the concatenations over the ranks of d_type, of d_payload with string_base added to '"' payloads and bytes_before to 'd'
 * payloads, and of d_strbuf[0, string_bytes), they are byte-identical to sjb200_tokens_dev on the whole document (whose
 * d_idx is the ranks' d_idx + bytes_before) when error is SUCCESS or a token error and short_ranks == 0.  Under CAPACITY
 * each rank did what sjb200_tokens_dev does on its shard with its own strbuf_capacity.
 *
 * finish returns, on every rank alike: UNEXPECTED_ERROR when dirty_cuts != 0, when a peer enqueued another kind for the
 * pass, or when a rank could not run its pass; else the error code of the first token in error in document order (the
 * earliest rank's first), with first_error_index; else CAPACITY when some rank is short; else SUCCESS -- the precedence
 * of sjb200_tokens_dev, where a token error wins over CAPACITY.  One host-synchronised round, no re-scan. */
typedef struct {
  int error;                  /* as returned */
  uint32_t dirty_cuts;        /* bit r: rank r entered its shard with state_in != 0 */
  uint32_t short_ranks;       /* bit r: rank r's string bytes exceed its strbuf_capacity (it wrote no records) */
  uint32_t reserved;
  uint64_t first_error_index; /* document-global structural index of the first token in error; UINT64_MAX if none */
  uint64_t tokens_before;     /* n of all earlier ranks: token k here is token tokens_before + k of the document */
  uint64_t bytes_before;      /* byte offset of this shard: a 'd' payload p is document offset bytes_before + p */
  uint64_t n_strings, strings_before, total_strings;
  uint64_t string_bytes, string_base, total_string_bytes; /* this rank's part of string_buf, its offset, the whole */
} sjb200_sharded_tokens_result;
SJB200_API int sjb200_tokens_sharded_enqueue(sjb200_comm *comm, const uint8_t *d_shard, size_t len, uint32_t state_in, const uint32_t *d_idx,
                                  uint32_t n, uint8_t *d_type, uint64_t *d_payload, uint8_t *d_strbuf, size_t strbuf_capacity, void *stream);
SJB200_API int sjb200_tokens_sharded_finish(sjb200_comm *comm, sjb200_sharded_tokens_result *out);
SJB200_API int sjb200_tokens_sharded(sjb200_comm *comm, const uint8_t *d_shard, size_t len, uint32_t state_in, const uint32_t *d_idx, uint32_t n,
                          uint8_t *d_type, uint64_t *d_payload, uint8_t *d_strbuf, size_t strbuf_capacity, sjb200_sharded_tokens_result *out,
                          void *stream);

/* stage-2 grammar (sjb200_document_errors_dev) sharded the same way, on the same comm and window: every rank judges its
 * own structurals, and three host-synchronised rounds carry what crosses the cuts -- the edges (each rank's n, table and
 * the types of its first two and last two structurals), the stack records (the containers open at each rank's end) and
 * the results (each rank's first error before its first document start, and its counts).  A grammar pass has its own
 * kind.  (d_type, d_payload, n) is this rank's output of sjb200_tokens_sharded; n may be 0.
 *   whole = 1: the ranks together hold ONE document, judged as dom::parser::parse judges it; d_docs / ndocs are ignored.
 *   whole = 0: d_docs / ndocs is this rank's table from sjb200_document_table_shard_dev (ndocs may be 0: a rank inside
 *              one long document).
 * Every rank passes the same whole and max_depth.  The contract: gather the inputs -- the concatenations of the ranks'
 * types, payloads, and tables with index + tokens_before -- and run sjb200_document_errors_dev on them.  Rank r writes
 * d_out[j] for the j-th document that STARTS on it (whole mode: rank 0 writes the one result), each {error, 64-bit
 * global structural index}; concatenated over the ranks they equal that call's d_out (whose 0xFFFFFFFF is UINT64_MAX
 * here).  The stream's structural 0 starts a segment whatever its rank's table says, as bit 0 does there.  One exception:
 * whole = 0 with no document on any rank writes nothing, reports 0 documents and returns SUCCESS.
 * finish returns, on every rank alike, the error code of that call: CAPACITY (nothing written) when a rank's max_depth
 * is 0 or above SJB200_DOCUMENT_MAX_DEPTH; UNEXPECTED_ERROR when any rank's table is bad (every result then
 * {UNEXPECTED_ERROR, UINT64_MAX}), when the ranks disagree on whole or max_depth, when a peer enqueued another kind for
 * the pass, or when a rank could not run its pass; else SUCCESS.  Deviations, as for sjb200_document_errors_dev: an
 * infinite float (1e400) is SUCCESS; a root token starting with a byte below '0' other than '-' (+1, #) is NUMBER_ERROR;
 * the last document wanting a value past the stream's end is a TAPE_ERROR at the global n. */
typedef struct {
  int32_t error;     /* simdjson::error_code */
  uint32_t reserved;
  uint64_t index;    /* global structural index at which it was decided (SUCCESS: one past the document's value); UINT64_MAX: none */
} sjb200_sharded_document_error;
typedef struct {
  int error;                    /* as returned */
  int32_t first_error;          /* the error of first_doc_in_error (SUCCESS when none) */
  uint64_t docs_before;         /* documents starting on earlier ranks: d_out[j] here is document docs_before + j */
  uint64_t tokens_before;       /* structurals of earlier ranks */
  uint64_t ndocs;               /* documents of the stream */
  uint64_t ndocs_in_error;
  uint64_t first_doc_in_error;  /* global document number; UINT64_MAX when none */
  uint64_t first_error_index;   /* its global structural index; UINT64_MAX when none */
} sjb200_sharded_document_errors_result;
SJB200_API int sjb200_document_errors_sharded_enqueue(sjb200_comm *comm, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, int whole,
                                                      const sjb200_doc_boundary *d_docs, uint32_t ndocs, size_t max_depth,
                                                      sjb200_sharded_document_error *d_out, void *stream);
SJB200_API int sjb200_document_errors_sharded_finish(sjb200_comm *comm, sjb200_sharded_document_errors_result *out);
SJB200_API int sjb200_document_errors_sharded(sjb200_comm *comm, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, int whole,
                                              const sjb200_doc_boundary *d_docs, uint32_t ndocs, size_t max_depth,
                                              sjb200_sharded_document_error *d_out, sjb200_sharded_document_errors_result *out, void *stream);

/* JSON Pointer lookup (sjb200_at_pointer_dev) sharded the same way, on the same comm and window: every rank walks the
 * documents that start on it, and a walk that reaches the end of a rank inside its document is handed, as a small
 * record, to the next rank that holds structurals, which resumes it.  A pointer pass has its own kind.  (d_type,
 * d_payload, n, d_strbuf, string_bytes) is this rank's output of sjb200_tokens_sharded; string payloads and d_strbuf stay
 * rank-local.  n may be 0.
 *   whole = 1: the ranks together hold ONE document; d_docs / ndocs are ignored.
 *   whole = 0: d_docs / ndocs is this rank's table from sjb200_document_table_shard_dev (ndocs may be 0: a rank inside
 *              one long document).
 * Every rank passes the same whole and the same pointers.  The contract: gather the inputs -- the concatenations of the
 * ranks' types, payloads ('"' payloads + string_base), string buffers and tables (index + tokens_before) -- and run
 * sjb200_at_pointer_dev on them (no table in whole mode).  Rank r's d_out[p * ndocs + j] (device memory) is that call's
 * result for pointer p and document docs_before + j, the j-th document that STARTS on rank r; in whole mode rank 0
 * writes the npointers results.  Indexes are global and 64-bit (0xFFFFFFFF there is UINT64_MAX here).  For a document
 * that spans ranks the first token in error is the first over all of its pieces.  Two exceptions: a bad table on any
 * rank makes every result {UNEXPECTED_ERROR, UINT64_MAX} (where a document on one rank ends depends on the others'
 * tables); whole = 0 with no document on any rank writes nothing, reports 0 documents and returns SUCCESS.
 * finish returns, on every rank alike: CAPACITY (nothing written) when a rank has more than
 * SJB200_POINTER_SHARDED_MAX_POINTERS pointers or is over a limit of sjb200_at_pointer_dev, or the stream has 2^32 - 3
 * structurals or more; UNEXPECTED_ERROR when a peer enqueued another kind for the pass, when a rank could not run its
 * pass, when the ranks disagree on whole or on the pointers (their count and a 64-bit hash of the compiled pointers), or
 * for a bad table; else SUCCESS.  Rounds: the edge round, then one round per step of the walks (the first step is the
 * local walks) until a step hands nothing over -- at most nranks of them, one when no walk crosses a cut.  The window
 * area is DESIGN.md section 5. */
#define SJB200_POINTER_SHARDED_MAX_POINTERS 1024   /* pointers per sharded call (window space) */
typedef struct {
  int32_t error;     /* simdjson::error_code */
  uint32_t reserved;
  uint64_t index;    /* global structural index of the selected value / of the first token in error; UINT64_MAX: none */
} sjb200_sharded_pointer_result;
typedef struct {
  int error;                 /* as returned */
  uint32_t rounds;           /* continuation steps this pass ran (0 when no walk crossed a cut) */
  uint64_t docs_before;      /* documents starting on earlier ranks: d_out[p * ndocs + j] here is document docs_before + j */
  uint64_t tokens_before;    /* structurals of earlier ranks */
  uint64_t ndocs;            /* documents of the stream (whole mode: 1) */
  uint64_t walks_forwarded;  /* (document, pointer) walks this rank handed to a later rank */
} sjb200_sharded_pointer_summary;
SJB200_API int sjb200_at_pointer_sharded_enqueue(sjb200_comm *comm, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                                 size_t string_bytes, int whole, const sjb200_doc_boundary *d_docs, uint32_t ndocs,
                                                 const char *const *pointers, const size_t *pointer_lens, int npointers,
                                                 sjb200_sharded_pointer_result *d_out, void *stream);
SJB200_API int sjb200_at_pointer_sharded_finish(sjb200_comm *comm, sjb200_sharded_pointer_summary *out);
SJB200_API int sjb200_at_pointer_sharded(sjb200_comm *comm, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                         size_t string_bytes, int whole, const sjb200_doc_boundary *d_docs, uint32_t ndocs, const char *const *pointers,
                                         const size_t *pointer_lens, int npointers, sjb200_sharded_pointer_result *d_out,
                                         sjb200_sharded_pointer_summary *out, void *stream);

/* the document starts of one shard of a sharded stream pass: (local structural index, shard-relative byte) pairs of
 * d_idx[0, kept), structural 0 counted when first_starts_document says so (both from the pass's result).  A rank's
 * global document numbers are its table's positions plus the other ranks' ndocs before it.  Not collective.
 * sjb200_document_table_dev is this call with first_starts_document = 1. */
SJB200_API int sjb200_document_table_shard_dev(sjb200_ctx *ctx, const uint8_t *d_shard, const uint32_t *d_idx, uint32_t kept, int first_starts_document,
                                    sjb200_doc_boundary *d_table, uint32_t capacity, uint32_t *ndocs_out, void *stream);

/* the host fold of the streaming round, pure (no device, no comm): what every rank's finish computes from the
 * nranks summaries.  Roles: 0 value, 1 ',' or ':', 2 '{', 3 '}', 4 '[', 5 ']'. */
typedef struct {
  uint64_t count;         /* in: structurals of the shard (after the second round) */
  uint32_t len;           /* shard length after the trim */
  uint32_t first_byte;    /* byte of structural 0 (count > 0) */
  uint32_t last_byte;     /* byte of structural count-1 (count > 0) */
  uint32_t start_index;   /* last document start >= 1 among the kept structurals (has_start) */
  uint32_t start_byte;
  int32_t net_obj;        /* '{' minus '}' from that start on, or over all kept structurals without one */
  int32_t net_arr;        /* '[' minus ']', likewise */
  uint32_t role_first;    /* role of the first kept structural */
  uint32_t role_last;     /* role of the last kept structural */
  uint32_t has_start;
} sjb200_stream_summary;
typedef struct {
  uint64_t kept;
  uint64_t bytes_before;
  uint32_t first_starts_document;
  uint32_t nrewrites;       /* 0..2 words of this rank's d_idx rewritten: d_idx[rewrite_pos[k]] = rewrite_val[k] */
  uint32_t rewrite_pos[2];
  uint32_t rewrite_val[2];
} sjb200_stream_rank;
typedef struct {
  int error;
  uint32_t n_written;       /* 0: n left untouched */
  uint64_t n;
  uint64_t total_bytes;
} sjb200_stream_fold_result;
/* final_state / flags_all as in sjb200_sharded_result.  Returns res->error. */
SJB200_API int sjb200_stream_fold(int mode, int nranks, uint32_t final_state, uint32_t flags_all, const sjb200_stream_summary *sums,
                       sjb200_stream_fold_result *res, sjb200_stream_rank *ranks /* nranks */);

/* the host fold of a delimited pass's filter round, pure: what every rank's finish computes.  Per shard: */
typedef struct {
  uint64_t count;         /* structurals of the shard's scan (after the second round) */
  uint32_t len;           /* shard length after the trim */
  uint32_t filtered;      /* entries its filter kept (with the carried-in depth / run) */
  uint32_t seps;          /* separators it counted: RS bytes of the runs of RS entries, or root commas */
  uint32_t last_sep;      /* shard-relative byte of the last one (seps > 0) */
  uint32_t below;         /* filtered entries before last_sep (seps > 0) */
  uint32_t reserved;
  sjb200_stream_summary walk;        /* the stream summary of the filtered entries (count is ignored) */
  sjb200_stream_summary walk_below;  /* the same of the first `below` of them (comma-delimited partial mode) */
} sjb200_delimited_summary;
typedef struct {
  uint64_t kept;
  uint64_t filtered_before;
  uint64_t bytes_before;
  uint32_t first_starts_document;
  uint32_t reserved;
} sjb200_delimited_rank;
typedef struct {
  int error;
  uint32_t n_written;       /* 0: n left untouched */
  uint64_t n;
  uint64_t total_bytes;
  /* the words n, n+1, n+2: tail_rank[k] < 0: the word is tail_val[k]; else rank tail_rank[k] holds it at local position
   * tail_pos[k] of its filtered entries (tail_filtered[k] = 1) or of its scanned structurals (0), shard-relative */
  int32_t tail_rank[3];
  uint32_t tail_pos[3];
  uint32_t tail_filtered[3];
  uint32_t tail_val[3];
} sjb200_delimited_fold_result;
SJB200_API int sjb200_delimited_fold(int mode, int nranks, uint32_t final_state, uint32_t flags_all, const sjb200_delimited_summary *sums,
                          sjb200_delimited_fold_result *res, sjb200_delimited_rank *ranks /* nranks */);

/* the host folds of a sharded grammar pass, pure: what every rank's finish computes.  The edge round, per rank: */
typedef struct {
  uint32_t n;            /* structurals */
  uint32_t ndocs;        /* table entries (whole mode: 0) */
  uint32_t flags;        /* bit0 the rank could not run its pass, bit1 bad table, bit2 whole, bit3 the table starts at 0,
                            bit4 its last entry is n - 1 */
  uint32_t max_depth;
  uint32_t types;        /* types of structurals 0, 1, n - 2, n - 1, a byte each from the low one (0xFF: none) */
  uint32_t first_start;  /* the table's first entry (ndocs > 0) */
} sjb200_grammar_edge;
typedef struct {
  uint64_t tokens_before;
  uint64_t docs_before;
  uint32_t owned;        /* documents that start on this rank (whole mode: 1 on rank 0) */
  uint32_t holds_root;   /* this rank's structural 0 is the stream's */
  uint32_t halo_before;  /* types of the two structurals before this rank's 0: byte 0 the earlier one (0xFF: none) */
  uint32_t halo_after;   /* type of the structural after this rank's last (0xFF: none) */
  uint32_t halo_flags;   /* bit0 the structural before this rank's 0 starts a document, bit1 the one after its last does,
                            bit2 holds_root */
  uint32_t last_type;    /* type of the stream's last structural (0xFF: none) */
} sjb200_grammar_rank;
typedef struct {
  int error;             /* SUCCESS, CAPACITY or UNEXPECTED_ERROR (a failed rank, whole / max_depth disagree) */
  uint32_t bad_table;    /* some rank's table is bad */
  uint64_t n;            /* structurals of the stream */
  uint64_t ndocs;        /* documents of the stream */
} sjb200_grammar_edge_fold_result;
SJB200_API int sjb200_grammar_edge_fold(int nranks, const sjb200_grammar_edge *edges, sjb200_grammar_edge_fold_result *res,
                                        sjb200_grammar_rank *ranks /* nranks */);
/* the result round, per rank: errors as keys global index << 8 | code (UINT64_MAX: none) */
typedef struct {
  uint64_t lead;         /* the first error among its structurals before its first document start */
  uint64_t last;         /* the first error its own structurals give its last document */
  uint64_t first_key;    /* that of first_doc */
  uint32_t errors;       /* its documents in error, the last one left out */
  uint32_t first_doc;    /* the first of them (0xFFFFFFFF: none) */
} sjb200_grammar_tally;
/* fills out's error, first_error, ndocs, ndocs_in_error, first_doc_in_error, first_error_index, and last[r], the result
 * of rank r's last document (ranks that own none: unchanged).  Returns out->error. */
SJB200_API int sjb200_grammar_result_fold(int nranks, const sjb200_grammar_edge *edges, const sjb200_grammar_tally *tallies,
                                          sjb200_sharded_document_errors_result *out, sjb200_sharded_document_error *last /* nranks */);

/* the host fold of a sharded pointer pass's edge round, pure: what every rank's finish computes.  Per rank: */
typedef struct {
  uint32_t n;            /* structurals */
  uint32_t ndocs;        /* table entries (whole mode: 0) */
  uint32_t flags;        /* bit0 the rank could not run its pass, bit1 bad table, bit2 whole, bit3 over a limit */
  uint32_t npointers;
  uint64_t hash;         /* of the compiled pointers */
  uint32_t types;        /* types of structurals 0 and n - 1, a byte each from the low one (0xFF: none) */
  uint32_t first_entry;  /* the table's first entry (n without one): structurals before it are the leading segment */
  uint32_t lead_error_index;  /* local index of the first token in error of the leading segment (0xFFFFFFFF: none) */
  uint32_t lead_error;        /* its error code */
} sjb200_pointer_edge;
typedef struct {
  uint64_t tokens_before;
  uint64_t docs_before;
  uint32_t owned;            /* results this rank writes: its table's documents (whole mode: 1 on rank 0) */
  uint32_t walks;            /* documents whose walks start here: owned, but in whole mode 1 on the first rank with n > 0 */
  int32_t prev_holder;       /* the last earlier rank with n > 0 (-1: none): it hands walks to this rank */
  int32_t next_holder;       /* the next later rank with n > 0 (-1: none) */
  uint32_t next_type;        /* type of the structural after this rank's last (0xFF: none) */
  int32_t lead_owner;        /* the rank whose document this rank's leading segment continues (-1: none) */
  int32_t tail_owner;        /* the rank whose document holds this rank's last structural (-1: none) */
  uint32_t tail_continues;   /* that document goes on past this rank */
  int32_t tail_through;      /* the last rank it reaches */
  uint32_t tail_error;       /* the first token in error of its pieces on later ranks (0: none) */
  uint64_t tail_after;       /* its structurals on later ranks */
  uint64_t tail_error_index; /* global index of that token (UINT64_MAX: none) */
} sjb200_pointer_rank;
typedef struct {
  int error;             /* SUCCESS, CAPACITY or UNEXPECTED_ERROR (a failed rank, whole / pointers disagree) */
  uint32_t bad_table;    /* some rank's table is bad (whole = 0; the pass then fails after writing its results) */
  uint64_t n;            /* structurals of the stream */
  uint64_t ndocs;        /* documents of the stream */
} sjb200_pointer_edge_fold_result;
SJB200_API int sjb200_pointer_edge_fold(int nranks, const sjb200_pointer_edge *edges, sjb200_pointer_edge_fold_result *res,
                                        sjb200_pointer_rank *ranks /* nranks */);

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
