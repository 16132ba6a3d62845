/*
 * sj_grammar_oracle.c -- CPU restatement of json_iterator::walk_document (src/generic/stage2/json_iterator.h L120-367)
 * with tape_builder, over stage-2-lite tokens (sjo_tokens output).  TEST INFRASTRUCTURE ONLY: the walk's own states, one
 * structural at a time with an explicit stack, so that it shares no structure with the device pass
 * (simdjson_b200/csrc/sjb200_grammar.cuh).  Recipe: oracle/grammar.mk.
 */
#include "sj_grammar_oracle.h"

#include <stdlib.h>

enum { TAPE_ERROR = 3, DEPTH_ERROR = 4, STRING_ERROR = 5, NUMBER_ERROR = 9, EMPTY = 13 };

static int is_scalar(uint8_t t) { return t == '"' || t == 'l' || t == 'u' || t == 'd' || t == 't' || t == 'f' || t == 'n'; }

/* visit_primitive / visit_root_primitive: what tape_builder returns for the token.  Inside a container every byte below
 * '0' takes the number path (json_iterator.h L342: `(*value - '0') < 10` in int), so a ',' there is a NUMBER_ERROR; the
 * root's switch (L309-336) sends it to TAPE_ERROR. */
static int visit_scalar(const uint8_t *type, const uint64_t *payload, uint32_t k, int root) {
  if (is_scalar(type[k])) return 0;
  if (type[k] == 0) return (int)(payload[k] & 0xFF);
  if (type[k] == ',' && !root) return NUMBER_ERROR;
  return TAPE_ERROR;
}
/* visit_key after the `*key != '"'` check: only a string token can fail as a key with its own error */
static int visit_key(const uint8_t *type, const uint64_t *payload, uint32_t k) {
  if (type[k] == '"') return 0;
  return type[k] == 0 && (payload[k] & 0xFF) == STRING_ERROR ? STRING_ERROR : TAPE_ERROR;
}

int sjo_walk_document(const uint8_t *type, const uint64_t *payload, uint32_t n, uint32_t start, uint32_t end, int whole, size_t max_depth,
                      uint32_t *index) {
  if (end > n) end = n;
  if (start >= end) {
    *index = start;
    return EMPTY;
  }
  uint8_t *is_array = (uint8_t *)calloc(max_depth + 2, 1);
  size_t depth = 0;
  int err = 0;
  uint32_t next = start, k;
#define FAIL(code, at) do { err = (code); *index = (at); goto out; } while (0)
/* advance(): reading the structural at the document's end is a TAPE_ERROR there */
#define ADVANCE(var) do { if (next >= end) FAIL(TAPE_ERROR, end); (var) = next++; } while (0)
#define PEEK_IS(c) (next < end && type[next] == (c))
#define TRY(at, expr) do { const int e_ = (expr); if (e_) FAIL(e_, at); } while (0)
  ADVANCE(k);
  if (whole) {
    if (type[k] == '{' && type[n - 1] != '}') FAIL(TAPE_ERROR, k);
    if (type[k] == '[' && type[n - 1] != ']') FAIL(TAPE_ERROR, k);
  }
  switch (type[k]) {
    case '{': if (PEEK_IS('}')) { next++; break; } goto object_begin;
    case '[': if (PEEK_IS(']')) { next++; break; } goto array_begin;
    default: TRY(k, visit_scalar(type, payload, k, 1)); break;
  }
  goto document_end;

object_begin:
  depth++;
  if (depth >= max_depth) FAIL(DEPTH_ERROR, k);
  is_array[depth] = 0;
  ADVANCE(k);
  if (type[k] != '"' && type[k] != 0) FAIL(TAPE_ERROR, k);
  TRY(k, visit_key(type, payload, k));
object_field:
  ADVANCE(k);
  if (type[k] != ':') FAIL(TAPE_ERROR, k);
  ADVANCE(k);
  switch (type[k]) {
    case '{': if (PEEK_IS('}')) { next++; break; } goto object_begin;
    case '[': if (PEEK_IS(']')) { next++; break; } goto array_begin;
    default: TRY(k, visit_scalar(type, payload, k, 0)); break;
  }
object_continue:
  ADVANCE(k);
  switch (type[k]) {
    case ',':
      ADVANCE(k);
      TRY(k, visit_key(type, payload, k));
      goto object_field;
    case '}': goto scope_end;
    default: FAIL(TAPE_ERROR, k);
  }

scope_end:
  depth--;
  if (depth == 0) goto document_end;
  if (is_array[depth]) goto array_continue;
  goto object_continue;

array_begin:
  depth++;
  if (depth >= max_depth) FAIL(DEPTH_ERROR, k);
  is_array[depth] = 1;
array_value:
  ADVANCE(k);
  switch (type[k]) {
    case '{': if (PEEK_IS('}')) { next++; break; } goto object_begin;
    case '[': if (PEEK_IS(']')) { next++; break; } goto array_begin;
    default: TRY(k, visit_scalar(type, payload, k, 0)); break;
  }
array_continue:
  ADVANCE(k);
  switch (type[k]) {
    case ',': goto array_value;
    case ']': goto scope_end;
    default: FAIL(TAPE_ERROR, k);
  }

document_end:
  /* a walk that ends before the document's end: the first structural left over (L237-240; parse_many: L332-334) */
  if (next < end) FAIL(TAPE_ERROR, next);
  *index = next;
  err = 0;
out:
#undef FAIL
#undef ADVANCE
#undef PEEK_IS
#undef TRY
  free(is_array);
  return err;
}

int sjo_document_errors(const uint8_t *type, const uint64_t *payload, uint32_t n, const uint32_t *starts, uint32_t ndocs, size_t max_depth,
                        int32_t *errors, uint32_t *indexes) {
  if (ndocs == 0 || starts == NULL) {
    if (n == 0) {
      errors[0] = EMPTY;
      indexes[0] = 0;
      return 1;
    }
    errors[0] = sjo_walk_document(type, payload, n, 0, n, 1, max_depth, indexes);
    return errors[0] != 0;
  }
  for (uint32_t d = 0; d < ndocs; d++)
    if (starts[d] >= n || (d > 0 && starts[d - 1] >= starts[d])) {
      for (uint32_t e = 0; e < ndocs; e++) {
        errors[e] = 24;
        indexes[e] = 0xFFFFFFFFu;
      }
      return (int)ndocs;
    }
  int bad = 0;
  for (uint32_t d = 0; d < ndocs; d++) {
    const uint32_t end = d + 1 < ndocs ? starts[d + 1] : n;
    errors[d] = sjo_walk_document(type, payload, n, starts[d], end, 0, max_depth, indexes + d);
    bad += errors[d] != 0;
  }
  return bad;
}
