// dropin_harness.cpp -- C entry points that drive the UNMODIFIED simdjson public API (dom::parser::parse,
// parse_many, ondemand::parser::iterate, simdjson::minify, simdjson::validate_utf8) with either the "b200"
// plug-in or a CPU implementation active, so the pytest drop-in tests can compare the two.  It is the
// reference-side usage a maintainer would write (INTEGRATION.md), wrapped for ctypes.
#include <chrono>
#include <cstring>
#include <memory>
#include <string>

#include "b200_implementation.h"

using namespace simdjson;

#define HARNESS_API extern "C" __attribute__((visibility("default")))

namespace {
const implementation *pick(int use_b200, int device) {
  if (use_b200) return b200::get_implementation(device);
  for (const char *n : {"icelake", "haswell", "westmere", "fallback"}) {
    auto impl = get_available_implementations()[n];
    if (impl && impl->supported_by_runtime_system()) return impl;
  }
  return builtin_implementation();
}
struct scoped_impl {
  const implementation *saved;
  explicit scoped_impl(const implementation *impl) : saved(get_active_implementation()) { get_active_implementation() = impl; }
  ~scoped_impl() { get_active_implementation() = saved; }
};
void put(const std::string &s, char *out, size_t cap, size_t *out_len) {
  *out_len = s.size();
  if (s.size() <= cap) std::memcpy(out, s.data(), s.size());
}

// Per-document records of the stream walks, serialised little-endian so that two walks compare as two byte strings:
// i32 fields, u64 fields, and byte fields as a u64 length followed by the bytes.  NONE as a length or a number stands
// for "not recorded"; OUT_OF_RANGE for a source() view that does not lie inside the input.
constexpr uint64_t NONE = ~uint64_t(0), OUT_OF_RANGE = ~uint64_t(0) - 1;
struct record_writer {
  std::string s;
  void i32(int v) { s.append(reinterpret_cast<const char *>(&v), 4); }
  void u64(uint64_t v) { s.append(reinterpret_cast<const char *>(&v), 8); }
  void bytes(std::string_view v) { u64(v.size()); s.append(v.data(), v.size()); }
  // it.source() as a view into the walked input [buf, buf + len)
  void source(std::string_view v, const char *buf, size_t len) {
    if (v.data() < buf || size_t(v.data() - buf) > len || v.size() > len - size_t(v.data() - buf)) u64(OUT_OF_RANGE);
    else bytes(v);
  }
};

// The input of a walk as a user would hold it: len bytes followed by SIMDJSON_PADDING bytes of pad_fill (not zeros, so a
// result cannot depend on them), after 64 bytes of '#'.  ondemand's source() of a scalar in a later batch measures from
// the wrong origin and trims whitespace backwards from there; the '#' bytes stop that scan inside this allocation.
struct walk_input {
  std::unique_ptr<char[]> storage;
  char *data;
  walk_input(const uint8_t *buf, size_t len, int pad_fill) : storage(new char[64 + len + SIMDJSON_PADDING]), data(storage.get() + 64) {
    std::memset(storage.get(), '#', 64);
    if (len) std::memcpy(data, buf, len);
    std::memset(data + len, pad_fill, SIMDJSON_PADDING);
  }
};

// 0 whitespace_delimited, 1 json_sequence, 2 comma_delimited, 3 comma_delimited_array
bool to_format(int format, stream_format *f) {
  switch (format) {
    case 0: *f = stream_format::whitespace_delimited; return true;
    case 1: *f = stream_format::json_sequence; return true;
    case 2: *f = stream_format::comma_delimited; return true;
    case 3: *f = stream_format::comma_delimited_array; return true;
    default: return false;
  }
}

// truncated_bytes() reads structural_indexes[n] and [n + 1].  Stage 1 leaves those words unspecified when it returns
// before writing its sentinels (json_structural_indexer.h L195-263).  A stream calls stage 1 in the streaming modes
// only, where that happens on unescaped characters and internal errors (an unclosed string is tolerated there, L255-256,
// so UNCLOSED_STRING can only come from stage 2, after the sentinels): after such an ending the value is recorded as
// NONE.  document_stream answers CAPACITY itself (len - batch_start) and an empty input never reaches stage 1's writes.
// A parser that could not allocate (UNSUPPORTED_ARCHITECTURE: no GPU) has no index array to read at all.
bool truncated_is_defined(error_code final_err, size_t len) {
  if (len == 0) return false;
  return !(final_err == UNESCAPED_CHARS || final_err == MEMALLOC || final_err == UNEXPECTED_ERROR || final_err == UNSUPPORTED_ARCHITECTURE ||
           final_err == UNINITIALIZED);
}

}  // namespace

HARNESS_API const char *dropin_active_name(int use_b200) {
  static thread_local std::string s;
  scoped_impl g(pick(use_b200, 0));
  s = get_active_implementation()->name();
  return s.c_str();
}

// the implementation simdjson would use right now (no override by the harness)
HARNESS_API const char *dropin_default_active_name() {
  static thread_local std::string s;
  s = get_active_implementation()->name();
  return s.c_str();
}

// dom::parser::parse -> simdjson::minify(element).  gpu_calls reports how many stage-1 calls the parser's
// implementation sent to the GPU (0 for a CPU implementation).
HARNESS_API int dropin_dom_roundtrip(int use_b200, const uint8_t *buf, size_t len, char *out, size_t cap, size_t *out_len,
                                     unsigned long long *gpu_calls) {
  scoped_impl g(pick(use_b200, 0));
  dom::parser parser;
  dom::element doc;
  auto err = parser.parse(buf, len, true).get(doc);
  *out_len = 0;
  if (gpu_calls) {
    auto *p = dynamic_cast<b200::dom_parser_implementation *>(parser.implementation.get());
    *gpu_calls = p ? p->gpu_stage1_calls() : 0;
  }
  if (err) return int(err);
  put(simdjson::minify(doc), out, cap, out_len);
  return 0;
}

// dom::parser::parse_many (document_stream; with SIMDJSON_THREADS_ENABLED its stage-1 worker runs a second
// parser concurrently): concatenated minified documents, '\n' separated.
HARNESS_API long dropin_parse_many(int use_b200, const uint8_t *buf, size_t len, size_t batch_size, char *out, size_t cap,
                                   size_t *out_len, int *first_err, unsigned long long *gpu_calls) {
  scoped_impl g(pick(use_b200, 0));
  long ndocs = 0;
  *first_err = 0;
  std::string acc;
  dom::parser parser;
  {
    dom::document_stream stream;
    auto err = parser.parse_many(buf, len, batch_size).get(stream);
    if (err) {
      *first_err = int(err);
    } else {
      for (auto it = stream.begin(); it != stream.end(); ++it) {
        auto doc = *it;
        if (doc.error()) { *first_err = int(doc.error()); break; }
        acc += simdjson::minify(doc.value_unsafe());
        acc.push_back('\n');
        ndocs++;
      }
    }
  }
  if (gpu_calls) {
    auto *p = dynamic_cast<b200::dom_parser_implementation *>(parser.implementation.get());
    *gpu_calls = p ? p->gpu_stage1_calls() : 0;
  }
  put(acc, out, cap, out_len);
  return ndocs;
}

// dom::parser::parse_many(buf, len, batch_size, format) walked to its end: per iterator position
//   i32 doc.error(), u64 current_index(), source() and simdjson::minify(doc) (both NONE when the position has an error),
// then the trailer
//   i32 error of parse_many itself, u64 records, i32 record cap hit, u64 truncated_bytes(), u64 size_in_bytes().
// The walk stops after max_records records and says so, rather than looping on a stream that never ends.  format is
// 0 whitespace_delimited, 1 json_sequence, 2 comma_delimited, 3 comma_delimited_array; threaded sets parser.threaded
// (the stage-1 worker then runs a second parser concurrently and swaps it with this one).  gpu_calls: stage-1 calls the
// walk sent to the GPU, its worker's included (kept out of the records so that they compare across implementations).
// Returns 0, or -1 for an unknown format; out_len is the size of the records even when they did not fit in cap.
HARNESS_API int dropin_stream_dom(int use_b200, const uint8_t *buf, size_t len, size_t batch_size, int format, int threaded, int pad_fill,
                                  size_t max_records, char *out, size_t cap, size_t *out_len, unsigned long long *gpu_calls) {
  stream_format fmt;
  *out_len = 0;
  if (!to_format(format, &fmt)) return -1;
  scoped_impl g(pick(use_b200, 0));
  const uint64_t calls0 = b200::gpu_stage1_calls_total();
  walk_input in(buf, len, pad_fill);
  record_writer w;
  dom::parser parser;
  parser.threaded = threaded != 0;
  uint64_t records = 0, truncated = NONE, size = NONE;
  int cap_hit = 0;
  error_code final_err = SUCCESS;
  dom::document_stream stream;
  const error_code create_err = parser.parse_many(in.data, len, batch_size, fmt).get(stream);
  if (!create_err) {
    for (auto it = stream.begin(); it != stream.end(); ++it) {
      if (records == max_records) { cap_hit = 1; break; }
      auto doc = *it;
      final_err = doc.error();
      w.i32(int(doc.error()));
      w.u64(it.current_index());
      if (doc.error()) {
        w.u64(NONE);
        w.u64(NONE);
      } else {
        w.source(it.source(), in.data, len);
        w.bytes(simdjson::minify(doc.value_unsafe()));
      }
      records++;
    }
    if (truncated_is_defined(final_err, len)) truncated = stream.truncated_bytes();
    size = stream.size_in_bytes();
  }
  w.i32(int(create_err));
  w.u64(records);
  w.i32(cap_hit);
  w.u64(truncated);
  w.u64(size);
  if (gpu_calls) *gpu_calls = b200::gpu_stage1_calls_total() - calls0;
  put(w.s, out, cap, out_len);
  return 0;
}

// ondemand::parser::iterate_many over the same padded input, walked the same way: per iterator position
//   i32 it.error(), u64 current_index(), source() (NONE with an error), i32 error of to_json_string(doc) and its text
//   (NONE with an error),
// then the trailer of dropin_stream_dom.  format 0-3 as there; 4 is the deprecated iterate_many(..., allow_comma_separated
// = true) overload.  source() is taken before the document is read, as the API asks.
HARNESS_API int dropin_stream_ondemand(int use_b200, const uint8_t *buf, size_t len, size_t batch_size, int format, int threaded,
                                       int pad_fill, size_t max_records, char *out, size_t cap, size_t *out_len,
                                       unsigned long long *gpu_calls) {
  stream_format fmt = stream_format::comma_delimited;
  *out_len = 0;
  if (format != 4 && !to_format(format, &fmt)) return -1;
  scoped_impl g(pick(use_b200, 0));
  const uint64_t calls0 = b200::gpu_stage1_calls_total();
  walk_input in(buf, len, pad_fill);
  record_writer w;
  ondemand::parser parser;
  parser.threaded = threaded != 0;
  uint64_t records = 0, truncated = NONE, size = NONE;
  int cap_hit = 0;
  error_code final_err = SUCCESS;
  ondemand::document_stream stream;
  const padded_string_view view(in.data, len, len + SIMDJSON_PADDING);
  error_code create_err;
  if (format == 4) {
    SIMDJSON_PUSH_DISABLE_WARNINGS
    SIMDJSON_DISABLE_DEPRECATED_WARNING
    create_err = parser.iterate_many(view, batch_size, true).get(stream);
    SIMDJSON_POP_DISABLE_WARNINGS
  } else {
    create_err = parser.iterate_many(view, batch_size, fmt).get(stream);
  }
  if (!create_err) {
    for (auto it = stream.begin(); it != stream.end(); ++it) {
      if (records == max_records) { cap_hit = 1; break; }
      auto doc = *it;
      final_err = it.error();
      w.i32(int(it.error()));
      w.u64(it.current_index());
      if (it.error()) {
        w.u64(NONE);
        w.i32(int(it.error()));
        w.u64(NONE);
      } else {
        w.source(it.source(), in.data, len);
        std::string_view sv;
        const error_code jerr = simdjson::to_json_string(doc).get(sv);
        w.i32(int(jerr));
        if (jerr) w.u64(NONE);
        else w.bytes(sv);
      }
      records++;
    }
    if (truncated_is_defined(final_err, len)) truncated = stream.truncated_bytes();
    size = stream.size_in_bytes();
  }
  w.i32(int(create_err));
  w.u64(records);
  w.i32(cap_hit);
  w.u64(truncated);
  w.u64(size);
  if (gpu_calls) *gpu_calls = b200::gpu_stage1_calls_total() - calls0;
  put(w.s, out, cap, out_len);
  return 0;
}

// One dom::parser parses bufs[0..count) in turn (parse(buf, len, true): the parser's own padded copy), as a service
// parsing one request after another would: per document i32 error and minify(doc) (NONE with an error).  With
// initial_capacity > 0 the parser first allocate()s that much, so a later, larger document makes it grow.
HARNESS_API int dropin_dom_sequence(int use_b200, const uint8_t *const *bufs, const size_t *lens, size_t count, size_t initial_capacity,
                                    char *out, size_t cap, size_t *out_len, unsigned long long *gpu_calls) {
  scoped_impl g(pick(use_b200, 0));
  const uint64_t calls0 = b200::gpu_stage1_calls_total();
  *out_len = 0;
  record_writer w;
  dom::parser parser;
  int rc = 0;
  if (initial_capacity > 0) rc = int(parser.allocate(initial_capacity));
  for (size_t i = 0; rc == 0 && i < count; i++) {
    dom::element doc;
    const error_code err = parser.parse(bufs[i], lens[i], true).get(doc);
    w.i32(int(err));
    if (err) w.u64(NONE);
    else w.bytes(simdjson::minify(doc));
  }
  if (gpu_calls) *gpu_calls = b200::gpu_stage1_calls_total() - calls0;
  put(w.s, out, cap, out_len);
  return rc;
}

// ondemand::parser::iterate -> to_json_string (On-Demand walks the GPU-produced index array lazily)
HARNESS_API int dropin_ondemand_roundtrip(int use_b200, const uint8_t *buf, size_t len, char *out, size_t cap, size_t *out_len) {
  scoped_impl g(pick(use_b200, 0));
  *out_len = 0;
  padded_string json(reinterpret_cast<const char *>(buf), len);
  ondemand::parser parser;
  ondemand::document doc;
  auto err = parser.iterate(json).get(doc);
  if (err) return int(err);
  std::string_view sv;
  err = simdjson::to_json_string(doc).get(sv);
  if (err) return int(err);
  put(std::string(sv), out, cap, out_len);
  return 0;
}

// the free functions simdjson::minify(buf,len,dst,dst_len) / simdjson::validate_utf8(buf,len)
HARNESS_API int dropin_minify(int use_b200, const uint8_t *buf, size_t len, uint8_t *dst, size_t *dst_len) {
  scoped_impl g(pick(use_b200, 0));
  size_t n = 0;
  auto err = simdjson::minify(reinterpret_cast<const char *>(buf), len, reinterpret_cast<char *>(dst), n);
  *dst_len = n;
  return int(err);
}

HARNESS_API int dropin_validate_utf8(int use_b200, const uint8_t *buf, size_t len) {
  scoped_impl g(pick(use_b200, 0));
  return simdjson::validate_utf8(reinterpret_cast<const char *>(buf), len) ? 1 : 0;
}

// Stage 1 alone through the reference's own boundary, timed inside the process: what `bench.py` reports as e2e.
// get_active_implementation()->create_dom_parser_implementation(...)->stage1(buf, len, regular) on a pageable
// padded_string (the memory dom::parser::parse hands its implementation), `iters` calls after two warm-up calls.
// Returns the error code of the last call; seconds[0] = total of the timed calls, seconds[1] = the fastest call.
// idx_out (optional, idx_cap words): the n + 3 index words of the last call, for the parity gate.
HARNESS_API int dropin_stage1_timed(int use_b200, const uint8_t *buf, size_t len, int iters, double *seconds, uint32_t *n_out,
                                    uint32_t *idx_out, size_t idx_cap, unsigned long long *gpu_calls) {
  scoped_impl g(pick(use_b200, 0));
  std::unique_ptr<internal::dom_parser_implementation> p;
  auto err = get_active_implementation()->create_dom_parser_implementation(len, 1024, p);
  if (err) return int(err);
  padded_string json(reinterpret_cast<const char *>(buf), len);
  const uint8_t *b = reinterpret_cast<const uint8_t *>(json.data());
  for (int i = 0; i < 2; i++) err = p->stage1(b, len, stage1_mode::regular);
  double total = 0, best = 1e30;
  for (int i = 0; i < iters; i++) {
    const auto t0 = std::chrono::steady_clock::now();
    err = p->stage1(b, len, stage1_mode::regular);
    const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    total += dt;
    if (dt < best) best = dt;
  }
  seconds[0] = total;
  seconds[1] = best;
  *n_out = p->n_structural_indexes;
  if (idx_out && size_t(p->n_structural_indexes) + 3 <= idx_cap) std::memcpy(idx_out, p->structural_indexes.get(), (size_t(p->n_structural_indexes) + 3) * 4);
  if (gpu_calls) {
    auto *bp = dynamic_cast<b200::dom_parser_implementation *>(p.get());
    *gpu_calls = bp ? bp->gpu_stage1_calls() : 0;
  }
  return int(err);
}
