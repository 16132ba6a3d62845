/*
 * sj_grammar_oracle.h -- CPU restatement of json_iterator::walk_document over stage-2-lite tokens (sjo_tokens output of
 * sj_oracle.h).  TEST INFRASTRUCTURE ONLY: nothing under oracle/ is linked, imported or executed by the product path.
 * Pinned to the reference by tests/test_document_errors_oracle.py (live, through oracle/ref_grammar_driver.cpp) and by
 * tests/golden/document_errors.json (generator: oracle/gen_golden_document_errors.py).
 */
#ifndef SJ_GRAMMAR_ORACLE_H
#define SJ_GRAMMAR_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The error stage 2 returns for the document at structurals [start, end) of sjo_tokens output, with *index the
 * structural at which it was decided (SUCCESS: one past the document's value).  whole = 1: dom::parser::parse of the
 * buffer (the document is [0, n), with the unmatched root-bracket check); 0: stage2_next started at `start`, where
 * reading the structural at `end` is a TAPE_ERROR at end and a walk that ends before end is a TAPE_ERROR at the first
 * structural left over.  start >= end: EMPTY. */
int sjo_walk_document(const uint8_t *type, const uint64_t *payload, uint32_t n, uint32_t start, uint32_t end, int whole, size_t max_depth,
                      uint32_t *index);

/* every document of a stream: starts / ndocs a document table (NULL or 0: one document, whole), results per document
 * (UNEXPECTED_ERROR, 0xFFFFFFFF for all when the table is not ascending or has an entry at or above n).  Returns the
 * documents in error. */
int sjo_document_errors(const uint8_t *type, const uint64_t *payload, uint32_t n, const uint32_t *starts, uint32_t ndocs, size_t max_depth,
                        int32_t *errors, uint32_t *indexes);

#ifdef __cplusplus
}
#endif
#endif
