// ref_double_driver.cpp -- a C entry point into the UNMODIFIED reference's dom::parser::parse, dom::element::at_pointer
// and element::get_double, compiled with the reference's singleheader sources where they lie (recipe: oracle/double.mk ->
// oracle/_ref/libsj_ref_double.so).  TEST INFRASTRUCTURE ONLY: the checker of oracle/sj_double_oracle.c.
#include "simdjson.h"

#include <cstring>
#include <string_view>

using namespace simdjson;

#define SJR_API extern "C" __attribute__((visibility("default")))

static const implementation *find_impl() {
  for (const char *n : {"icelake", "haswell", "westmere", "fallback"}) {
    auto impl = get_available_implementations()[n];
    if (impl && impl->supported_by_runtime_system()) return impl;
  }
  return nullptr;
}

// dom::parser::parse(buf, len) once, then for pointer k (the next lens[k] bytes of `pointers`) at_pointer and
// get_double: errs[k] (the parse error when parse failed, else at_pointer's, else get_double's) and bits[k] (the
// double's bits, 0 on an error).  Returns the parse error, -1 without an implementation.
SJR_API int sjr_dom_double(const uint8_t *buf, size_t len, const char *pointers, const size_t *lens, int np, int *errs, uint64_t *bits) {
  auto impl = find_impl();
  if (!impl) return -1;
  const implementation *saved = get_active_implementation();
  get_active_implementation() = impl;
  dom::parser parser;
  dom::element doc;
  auto err = parser.parse(buf, len, true).get(doc);
  for (int k = 0; k < np; k++) {
    errs[k] = int(err);
    bits[k] = 0;
    std::string_view p(pointers, lens[k]);
    pointers += lens[k];
    if (err) continue;
    dom::element v;
    error_code e = doc.at_pointer(p).get(v);
    double d = 0;
    if (!e) e = v.get_double().get(d);
    if (!e) std::memcpy(&bits[k], &d, 8);
    errs[k] = int(e);
  }
  get_active_implementation() = saved;
  return int(err);
}
