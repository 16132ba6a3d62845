/*
 * sj_column_oracle.h -- CPU restatement of the DOM getters on one JSON Pointer result over stage-2-lite tokens (sjo_tokens
 * output of sj_oracle.h; rows of sjo_at_pointer, sj_pointer_oracle.h): what sjb200_column_dev computes per row.
 * TEST INFRASTRUCTURE ONLY: nothing under oracle/ is linked, imported or executed by the product path.  Pinned to the
 * reference by tests/test_column_oracle.py (live, through oracle/ref_column_driver.cpp) and by tests/golden/columns.json
 * (generator: oracle/gen_golden_columns.py).
 */
#ifndef SJ_COLUMN_ORACLE_H
#define SJ_COLUMN_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* kinds: 1 get_int64, 2 get_uint64, 3 get_bool, 4 get_string, 5 get_array().size(), 6 get_object().size() */
enum { SJC_INT64 = 1, SJC_UINT64 = 2, SJC_BOOL = 3, SJC_STRING = 4, SJC_ARRAY_SIZE = 5, SJC_OBJECT_SIZE = 6 };

/* The getter `kind` on the row {row_error, row_index}: returns the error (a row in error keeps it; an index >= n, at a
 * token that is not a value, or -- STRING -- at a string whose record does not lie in [0, string_bytes) is
 * UNEXPECTED_ERROR 24), *row_type the value's type char (0 for those), *value the integer, 0 / 1 or the size (0 on an
 * error), and for STRING *str_off / *str_len the string's bytes in strbuf (0 / 0 on an error). */
int sjo_column(int kind, const uint8_t *type, const uint64_t *payload, uint32_t n, const uint8_t *strbuf, size_t string_bytes, int32_t row_error,
               uint32_t row_index, uint8_t *row_type, uint64_t *value, uint64_t *str_off, uint32_t *str_len);

#ifdef __cplusplus
}
#endif
#endif
