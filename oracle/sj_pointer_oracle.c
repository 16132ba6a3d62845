/*
 * sj_pointer_oracle.c -- CPU restatement of dom::element::at_pointer over stage-2-lite tokens (sjo_tokens output).
 * TEST INFRASTRUCTURE ONLY, like sj_oracle.c: recursive and one structural at a time, so that it shares no structure
 * with the device walk (simdjson_b200/csrc/sjb200_pointer.cuh).  Recipe: oracle/pointer.mk.
 */
#include "sj_pointer_oracle.h"

#include <string.h>
/* ---- JSON Pointer: dom::element::at_pointer restated over sjo_tokens output, recursively and one structural at a time
 * (include/simdjson/dom/element-inl.h L410-446, object-inl.h L104-147 and L246-254, array-inl.h L94-121 and L216-224,
 * jsonpathutil.h L20-50). */
typedef struct {
  const uint8_t *type;
  const uint64_t *payload;
  const uint8_t *strbuf;
  size_t string_bytes;
  uint32_t end;
} ptr_doc;

/* one past the value at k: a container's matching close, found by counting brackets */
static uint32_t ptr_skip(const ptr_doc *d, uint32_t k) {
  if (d->type[k] != '{' && d->type[k] != '[') return k + 1;
  int depth = 0;
  for (uint32_t i = k; i < d->end; i++) {
    const uint8_t t = d->type[i];
    if (t == '{' || t == '[') depth++;
    if ((t == '}' || t == ']') && --depth == 0) return i + 1;
  }
  return d->end;
}

static int ptr_well_formed(const char *p, size_t len) {
  if (len == 0 || p[0] != '/') return 0;
  const char *e = memchr(p, '~', len);
  if (!e) return 1;
  const size_t at = (size_t)(e - p);
  return at + 1 < len && (p[at + 1] == '0' || p[at + 1] == '1');
}

/* the escaped token t[0, tl) against the string record at offset off, unescaping ~0 and ~1 as it goes */
static int ptr_key_equals(const ptr_doc *d, uint64_t off, const char *t, size_t tl) {
  if (off + 4 > d->string_bytes) return 0;
  const uint8_t *r = d->strbuf + off;
  const uint64_t rl = (uint64_t)r[0] | ((uint64_t)r[1] << 8) | ((uint64_t)r[2] << 16) | ((uint64_t)r[3] << 24);
  if (off + 4 + rl > d->string_bytes) return 0;
  uint64_t j = 0;
  for (size_t i = 0; i < tl; i++, j++) {
    char c = t[i];
    if (c == '~') c = t[++i] == '0' ? '~' : '/';
    if (j >= rl || r[4 + j] != (uint8_t)c) return 0;
  }
  return j == rl;
}

static int ptr_walk(const ptr_doc *d, uint32_t v, const char *p, size_t len, uint32_t *index) {
  const uint8_t t = d->type[v];
  if (t != '{' && t != '[') {
    if (len) return ptr_well_formed(p, len) ? SJP_NO_SUCH_FIELD : SJP_INVALID_JSON_POINTER;
    *index = v;
    return SJP_SUCCESS;
  }
  if (len == 0) {
    *index = v;
    return SJP_SUCCESS;
  }
  if (p[0] != '/') return SJP_INVALID_JSON_POINTER;
  p++;
  len--;
  const char *slash = memchr(p, '/', len);
  const size_t tl = slash ? (size_t)(slash - p) : len;
  uint32_t child = 0xFFFFFFFFu;
  if (t == '{') {
    for (size_t i = 0; i < tl; i++)
      if (p[i] == '~') {
        if (i + 1 >= tl || (p[i + 1] != '0' && p[i + 1] != '1')) return SJP_INVALID_JSON_POINTER;
        i++;
      }
    for (uint32_t k = v + 1; k + 2 < d->end && d->type[k] != '}';) { /* key ':' value [','] */
      if (d->type[k] == '"' && ptr_key_equals(d, d->payload[k], p, tl)) {
        child = k + 2;
        break;
      }
      k = ptr_skip(d, k + 2);
      if (k < d->end && d->type[k] == ',') k++;
    }
    if (child == 0xFFFFFFFFu) return SJP_NO_SUCH_FIELD;
  } else {
    if (len == 1 && p[0] == '-') return SJP_INDEX_OUT_OF_BOUNDS;
    uint64_t want = 0;
    for (size_t i = 0; i < tl; i++) {
      const uint8_t digit = (uint8_t)(p[i] - '0');
      if (digit > 9) return SJP_INCORRECT_TYPE;
      if (i > 0 && p[0] == '0') return SJP_INVALID_JSON_POINTER;
      if (want > (UINT64_MAX - digit) / 10) return SJP_INDEX_OUT_OF_BOUNDS;
      want = want * 10 + digit;
    }
    if (tl == 0) return SJP_INVALID_JSON_POINTER;
    uint64_t ord = 0;
    for (uint32_t k = v + 1; k < d->end && d->type[k] != ']'; ord++) {
      if (ord == want) {
        child = k;
        break;
      }
      k = ptr_skip(d, k);
      if (k < d->end && d->type[k] == ',') k++;
    }
    if (child == 0xFFFFFFFFu) return SJP_INDEX_OUT_OF_BOUNDS;
  }
  if (child >= d->end) return t == '{' ? SJP_NO_SUCH_FIELD : SJP_INDEX_OUT_OF_BOUNDS;
  if (!slash) {
    *index = child;
    return SJP_SUCCESS;
  }
  return ptr_walk(d, child, slash, len - tl, index);
}

int sjo_at_pointer(const uint8_t *type, const uint64_t *payload, uint32_t n, const uint8_t *strbuf, size_t string_bytes, uint32_t root, uint32_t end,
                   const char *pointer, size_t len, uint32_t *index) {
  *index = 0xFFFFFFFFu;
  if (end > n) end = n;
  if (root >= end) return SJP_UNEXPECTED_ERROR;
  for (uint32_t k = root; k < end; k++)
    if (type[k] == 0) {
      *index = k;
      return (int)payload[k];
    }
  const ptr_doc d = {type, payload, strbuf, string_bytes, end};
  return ptr_walk(&d, root, pointer, len, index);
}
