/*
 * sj_pointer_oracle.h -- CPU restatement of dom::element::at_pointer over stage-2-lite tokens (sjo_tokens output of
 * sj_oracle.h).  TEST INFRASTRUCTURE ONLY: nothing under oracle/ is linked, imported or executed by the product path.
 * Pinned to the reference by tests/test_pointer_oracle.py (live, through oracle/ref_pointer_driver.cpp) and by
 * tests/golden/pointers.json (generator: oracle/gen_golden_pointers.py).
 */
#ifndef SJ_POINTER_ORACLE_H
#define SJ_POINTER_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* numeric values of simdjson::error_code (include/simdjson/error.h L19-54) */
enum {
  SJP_SUCCESS = 0,
  SJP_INCORRECT_TYPE = 17,
  SJP_INDEX_OUT_OF_BOUNDS = 19,
  SJP_NO_SUCH_FIELD = 20,
  SJP_INVALID_JSON_POINTER = 22,
  SJP_UNEXPECTED_ERROR = 24
};

/* dom::element::at_pointer of one document, structurals [root, end) of sjo_tokens output (strbuf: string_bytes in use):
 * the first token in error in the document wins ({its error code, *index = its structural index}); else the error
 * at_pointer returns with *index = 0xFFFFFFFF, or SUCCESS with *index = the structural index of the selected value.
 * root >= min(end, n): UNEXPECTED_ERROR. */
int sjo_at_pointer(const uint8_t *type, const uint64_t *payload, uint32_t n, const uint8_t *strbuf, size_t string_bytes, uint32_t root, uint32_t end,
                   const char *pointer, size_t len, uint32_t *index);

#ifdef __cplusplus
}
#endif
#endif
