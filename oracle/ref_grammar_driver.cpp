// ref_grammar_driver.cpp -- C entry points into the UNMODIFIED reference's stage 2, compiled with the reference's
// singleheader sources where they lie (recipe: oracle/grammar.mk -> oracle/_ref/libsj_ref_grammar.so).
// TEST INFRASTRUCTURE ONLY: the checker of oracle/sj_grammar_oracle.c.
#include "simdjson.h"

#include <cstring>

using namespace simdjson;

#define SJR_API extern "C" __attribute__((visibility("default")))

static const implementation *find_impl(const char *name) {
  if (name == nullptr || name[0] == 0) {
    for (const char *n : {"icelake", "haswell", "westmere", "fallback"}) {
      auto impl = get_available_implementations()[n];
      if (impl && impl->supported_by_runtime_system()) return impl;
    }
    return nullptr;
  }
  auto impl = get_available_implementations()[name];
  if (!impl || !impl->supported_by_runtime_system()) return nullptr;
  return impl;
}

SJR_API int sjr_grammar_supported(const char *name) { return find_impl(name) != nullptr; }

// dom::parser::parse(buf, len) with max_depth: its error code
SJR_API int sjr_parse_error(const char *name, const uint8_t *buf, size_t len, size_t max_depth) {
  auto impl = find_impl(name);
  if (!impl) return -1;
  const implementation *saved = get_active_implementation();
  get_active_implementation() = impl;
  dom::parser parser(len + 64);
  int err = int(parser.allocate(len + 64, max_depth));
  if (!err) {
    dom::element doc;
    err = int(parser.parse(buf, len, true).get(doc));
  }
  get_active_implementation() = saved;
  return err;
}

// Every document of a stream as document_stream judges it (include/simdjson/dom/document_stream-inl.h L250-269): one
// stage 1 over a zero-padded copy in `mode` (a stage1_mode: streaming_final as document_stream runs it; regular keeps
// the last documents that streaming_final drops when they are incomplete), then for each table start `starts[d]`,
// stage2_next from there.
// errors[d] = its error code; on SUCCESS, next_index[d] = the parser's next_structural_index after it (else
// 0xFFFFFFFF).  Returns stage 1's error, or -1.
SJR_API int sjr_stream_errors(const char *name, const uint8_t *buf, size_t len, int mode, size_t max_depth, const uint32_t *starts, uint32_t ndocs,
                              int *errors, uint32_t *next_index, uint32_t *n_out) {
  auto impl = find_impl(name);
  if (!impl) return -1;
  std::unique_ptr<internal::dom_parser_implementation> p;
  if (impl->create_dom_parser_implementation(len + 64, max_depth, p)) return -1;
  padded_string copy(reinterpret_cast<const char *>(buf), len);
  dom::document doc;
  if (doc.allocate(len + 64)) return -1;
  const int e1 = int(p->stage1(reinterpret_cast<const uint8_t *>(copy.data()), len, stage1_mode(mode)));
  *n_out = p->n_structural_indexes;
  if (e1) return e1;
  for (uint32_t d = 0; d < ndocs; d++) {
    p->next_structural_index = starts[d];
    errors[d] = int(p->stage2_next(doc));
    next_index[d] = errors[d] == 0 ? p->next_structural_index : 0xFFFFFFFFu;
  }
  return 0;
}
