// ref_column_driver.cpp -- a C entry point into the UNMODIFIED reference's dom::element::at_pointer followed by one DOM
// getter, compiled with the reference's singleheader sources where they lie (recipe: oracle/column.mk ->
// oracle/_ref/libsj_ref_column.so).  TEST INFRASTRUCTURE ONLY: the checker of oracle/sj_column_oracle.c.
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

// dom::parser::parse(buf, len) once, then for pointer k (the next lens[k] bytes of `pointers`) at_pointer and the getter
// `kind` (1 get_int64, 2 get_uint64, 3 get_bool, 4 get_string, 5 get_array().size(), 6 get_object().size()): errs[k]
// (the parse error when parse failed, else at_pointer's, else the getter's), values[k] (the value's bits, 0 / 1, the
// size; 0 on an error) and for get_string the bytes, one string after the other into `out`, out_lens[k] each (what does
// not fit out_cap is left out and its length still counted).  Returns the parse error, -1 without an implementation.
SJR_API int sjr_dom_column(const uint8_t *buf, size_t len, const char *pointers, const size_t *lens, int np, int kind, int *errs, uint64_t *values,
                           char *out, size_t out_cap, size_t *out_lens) {
  auto impl = find_impl();
  if (!impl) return -1;
  const implementation *saved = get_active_implementation();
  get_active_implementation() = impl;
  dom::parser parser;
  dom::element doc;
  auto err = parser.parse(buf, len, true).get(doc);
  size_t used = 0;
  for (int k = 0; k < np; k++) {
    errs[k] = int(err);
    values[k] = 0;
    out_lens[k] = 0;
    std::string_view p(pointers, lens[k]);
    pointers += lens[k];
    if (err) continue;
    dom::element v;
    error_code e = doc.at_pointer(p).get(v);
    if (!e) {
      switch (kind) {
        case 1: { int64_t x = 0; e = v.get_int64().get(x); if (!e) values[k] = uint64_t(x); break; }
        case 2: { uint64_t x = 0; e = v.get_uint64().get(x); if (!e) values[k] = x; break; }
        case 3: { bool x = false; e = v.get_bool().get(x); if (!e) values[k] = x ? 1 : 0; break; }
        case 4: {
          std::string_view s;
          e = v.get_string().get(s);
          if (!e) {
            out_lens[k] = s.size();
            if (used + s.size() <= out_cap) std::memcpy(out + used, s.data(), s.size());
            used += s.size();
          }
          break;
        }
        case 5: { dom::array a; e = v.get_array().get(a); if (!e) values[k] = a.size(); break; }
        case 6: { dom::object o; e = v.get_object().get(o); if (!e) values[k] = o.size(); break; }
        default: e = UNEXPECTED_ERROR;
      }
    }
    errs[k] = int(e);
  }
  get_active_implementation() = saved;
  return int(err);
}
