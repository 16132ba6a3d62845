/* sj_double_oracle.c -- CPU restatement of element::get_double on one JSON Pointer result over stage-2-lite tokens (the
 * row of sjb200_column_double_dev): the tape type says what the value is; a 'd' value is strtod of its text (glibc's
 * strtod rounds correctly) and NUMBER_ERROR when that is infinite; 'l' / 'u' are the casts double(int64) /
 * double(uint64).  TEST INFRASTRUCTURE ONLY: nothing under oracle/ is linked, imported or executed by the product path.
 * Pinned to the reference by tests/test_double_oracle.py (live, through oracle/ref_double_driver.cpp) and by
 * tests/golden/doubles.json (generator: oracle/gen_golden_doubles.py). */
#define _GNU_SOURCE
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { NUMBER_ERROR = 9, INCORRECT_TYPE = 17, UNEXPECTED_ERROR = 24 };

static int is_value(uint8_t t) {
  return t == '{' || t == '[' || t == '"' || t == 'l' || t == 'u' || t == 'd' || t == 't' || t == 'f' || t == 'n';
}

/* The row {row_error, row_index} over tokens (type, payload, n) of the input buf[0, len) with structurals idx: returns the
 * error (a row in error keeps it; an index >= n, at a token that is not a value, or at a 'd' whose span
 * [idx[k], payload[k]) is empty or not inside [0, len) is UNEXPECTED_ERROR 24), *row_type the type char (0 for those) and
 * *bits the double's bits (0 on an error). */
int sjo_double(const uint8_t *type, const uint64_t *payload, uint32_t n, const uint8_t *buf, size_t len, const uint32_t *idx, int32_t row_error,
               uint32_t row_index, uint8_t *row_type, uint64_t *bits) {
  *row_type = 0;
  *bits = 0;
  if (row_error != 0) return row_error;
  if (row_index >= n || !is_value(type[row_index])) return UNEXPECTED_ERROR;
  const uint8_t t = type[row_index];
  const uint64_t v = payload[row_index];
  double d;
  *row_type = t;
  if (t == 'l') {
    d = (double)(int64_t)v;
  } else if (t == 'u') {
    d = (double)v;
  } else if (t == 'd') {
    const uint64_t s = idx[row_index];
    if (!(s < v && v <= len)) { *row_type = 0; return UNEXPECTED_ERROR; }
    char *text = malloc(v - s + 1);
    if (!text) { *row_type = 0; return UNEXPECTED_ERROR; }
    memcpy(text, buf + s, v - s);
    text[v - s] = 0;
    d = strtod(text, NULL);
    free(text);
    if (isinf(d)) return NUMBER_ERROR;
  } else {
    return INCORRECT_TYPE;
  }
  memcpy(bits, &d, 8);
  return 0;
}
