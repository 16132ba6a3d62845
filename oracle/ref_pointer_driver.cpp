// ref_pointer_driver.cpp -- a C entry point into the UNMODIFIED reference's dom::element::at_pointer, compiled with the
// reference's singleheader sources where they lie (recipe: oracle/pointer.mk -> oracle/_ref/libsj_ref_pointer.so).
// TEST INFRASTRUCTURE ONLY: the checker of oracle/sj_pointer_oracle.c.
#include "simdjson.h"

#include <cstring>
#include <string>
#include <string_view>

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

SJR_API int sjr_pointer_supported(const char *name) { return find_impl(name) != nullptr; }

// dom::element::at_pointer on the root of dom::parser::parse(buf, len), for np pointers (pointer k: the next lens[k] bytes
// of `pointers`) on one parse: returns the parse error; errs[k] = at_pointer's error (the parse error when parse failed),
// and on success the selected element serialised with simdjson::minify goes to `out`, one after the other, out_lens[k]
// bytes each (0 on an error; what does not fit out_cap is left out and its length still counted).
SJR_API int sjr_dom_at_pointer(const char *name, const uint8_t *buf, size_t len, const char *pointers, const size_t *lens, int np, int *errs, char *out,
                               size_t out_cap, size_t *out_lens) {
  auto impl = find_impl(name);
  if (!impl) return -1;
  const implementation *saved = get_active_implementation();
  get_active_implementation() = impl;
  dom::parser parser;
  dom::element doc;
  auto err = parser.parse(buf, len, true).get(doc);
  size_t used = 0;
  for (int k = 0; k < np; k++) {
    out_lens[k] = 0;
    errs[k] = int(err);
    if (!err) {
      dom::element v;
      auto e = doc.at_pointer(std::string_view(pointers, lens[k])).get(v);
      errs[k] = int(e);
      if (!e) {
        std::string s = simdjson::minify(v);
        out_lens[k] = s.size();
        if (used + s.size() <= out_cap) std::memcpy(out + used, s.data(), s.size());
        used += s.size();
      }
    }
    pointers += lens[k];
  }
  get_active_implementation() = saved;
  return int(err);
}
