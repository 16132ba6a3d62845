/* sj_column_oracle.c -- see sj_column_oracle.h.  The getters of include/simdjson/dom/element-inl.h (get_int64,
 * get_uint64, get_bool, get_string) and the tape's scope count (src/generic/stage2/tape_builder.h, saturated at
 * 0xFFFFFF), restated one row at a time over the tokens. */
#include "sj_column_oracle.h"

enum { INCORRECT_TYPE = 17, NUMBER_OUT_OF_RANGE = 18, UNEXPECTED_ERROR = 24 };

static int is_value(uint8_t t) {
  return t == '{' || t == '[' || t == '"' || t == 'l' || t == 'u' || t == 'd' || t == 't' || t == 'f' || t == 'n';
}

/* the children of the container opened at structural k, counted one structural after the other up to its close or n */
static uint64_t scope_count(const uint8_t *type, uint32_t n, uint32_t k, int obj) {
  uint64_t count = 0;
  long depth = 0;
  for (uint64_t j = (uint64_t)k + 1; j < n; j++) {
    const uint8_t t = type[j];
    if (depth == 0) {
      if (t == '}' || t == ']') break;
      if (obj ? (t == '"' && j + 1 < n && type[j + 1] == ':') : (t != ','))
        count++;
    }
    if (t == '{' || t == '[') depth++;
    if (t == '}' || t == ']') depth--;
  }
  return count > 0xFFFFFF ? 0xFFFFFF : count;
}

int sjo_column(int kind, const uint8_t *type, const uint64_t *payload, uint32_t n, const uint8_t *strbuf, size_t string_bytes, int32_t row_error,
               uint32_t row_index, uint8_t *row_type, uint64_t *value, uint64_t *str_off, uint32_t *str_len) {
  *row_type = 0;
  *value = 0;
  *str_off = 0;
  *str_len = 0;
  if (row_error != 0) return row_error;
  if (row_index >= n || !is_value(type[row_index])) return UNEXPECTED_ERROR;
  const uint8_t t = type[row_index];
  const uint64_t v = payload[row_index];
  *row_type = t;
  switch (kind) {
    case SJC_INT64:
      if (t == 'l') { *value = v; return 0; }
      if (t == 'u') {
        if (v > (uint64_t)INT64_MAX) return NUMBER_OUT_OF_RANGE;
        *value = v;
        return 0;
      }
      return INCORRECT_TYPE;
    case SJC_UINT64:
      if (t == 'u') { *value = v; return 0; }
      if (t == 'l') {
        if ((int64_t)v < 0) return NUMBER_OUT_OF_RANGE;
        *value = v;
        return 0;
      }
      return INCORRECT_TYPE;
    case SJC_BOOL:
      if (t == 't') { *value = 1; return 0; }
      if (t == 'f') return 0;
      return INCORRECT_TYPE;
    case SJC_STRING: {
      if (t != '"') return INCORRECT_TYPE;
      if (v > string_bytes || string_bytes - v < 5) { *row_type = 0; return UNEXPECTED_ERROR; }
      const uint8_t *r = strbuf + v;
      const uint32_t len = (uint32_t)r[0] | ((uint32_t)r[1] << 8) | ((uint32_t)r[2] << 16) | ((uint32_t)r[3] << 24);
      if (string_bytes - v - 5 < len) { *row_type = 0; return UNEXPECTED_ERROR; }
      *str_off = v + 4;
      *str_len = len;
      return 0;
    }
    case SJC_ARRAY_SIZE:
      if (t != '[') return INCORRECT_TYPE;
      *value = scope_count(type, n, row_index, 0);
      return 0;
    case SJC_OBJECT_SIZE:
      if (t != '{') return INCORRECT_TYPE;
      *value = scope_count(type, n, row_index, 1);
      return 0;
    default:
      *row_type = 0;
      return UNEXPECTED_ERROR;
  }
}
