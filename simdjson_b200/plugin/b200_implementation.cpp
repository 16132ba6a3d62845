// b200_implementation.cpp -- see b200_implementation.h
#include "b200_implementation.h"

#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>

namespace simdjson {
namespace b200 {

namespace {

// The concrete class of the built-in CPU implementation (include/simdjson/generic/dom_parser_implementation.h
// L21-50): stage 2 reads its public `buf` / `len` members, so the inner parser is addressed by its real type.
using builtin_parser = simdjson::SIMDJSON_BUILTIN_IMPLEMENTATION::dom_parser_implementation;

inline error_code to_error(int rc) noexcept { return static_cast<error_code>(rc); }

// a lazily created context for the stateless implementation::minify / validate_utf8 calls, one per
// calling thread (the reference's are const and callable concurrently from any thread)
struct thread_context {
  sjb200_ctx *ctx{nullptr};
  int device{-1};
  ~thread_context() { if (ctx) sjb200_destroy(ctx); }
  sjb200_ctx *get(int dev) noexcept {
    if (ctx && device != dev) { sjb200_destroy(ctx); ctx = nullptr; }
    if (!ctx) { if (sjb200_create(dev, 0, &ctx) != SJB200_SUCCESS) ctx = nullptr; device = dev; }
    return ctx;
  }
};
thread_local thread_context tls_context;

std::atomic<uint64_t> total_gpu_calls{0};

}  // namespace

uint64_t gpu_stage1_calls_total() noexcept { return total_gpu_calls.load(); }

// ---------------------------------------------------------------- implementation
error_code implementation::create_dom_parser_implementation(size_t capacity, size_t max_depth,
                                                            std::unique_ptr<internal::dom_parser_implementation> &dst) const noexcept {
  dst.reset(new (std::nothrow) dom_parser_implementation(device_));
  if (!dst) return MEMALLOC;
  if (auto err = dst->set_capacity(capacity)) { dst.reset(); return err; }
  if (auto err = dst->set_max_depth(max_depth)) { dst.reset(); return err; }
  return SUCCESS;
}

error_code implementation::minify(const uint8_t *buf, size_t len, uint8_t *dst, size_t &dst_len) const noexcept {
  sjb200_ctx *ctx = tls_context.get(device_);
  if (!ctx) { dst_len = 0; return UNSUPPORTED_ARCHITECTURE; }
  size_t n = 0;
  const int rc = sjb200_minify(ctx, buf, len, dst, &n);
  dst_len = n;
  return to_error(rc);
}

bool implementation::validate_utf8(const char *buf, size_t len) const noexcept {
  sjb200_ctx *ctx = tls_context.get(device_);
  if (!ctx) return false;
  return sjb200_validate_utf8(ctx, reinterpret_cast<const uint8_t *>(buf), len) == 1;
}

const implementation *get_implementation(int device) noexcept {
  static implementation singletons[8] = {implementation(0), implementation(1), implementation(2), implementation(3),
                                         implementation(4), implementation(5), implementation(6), implementation(7)};
  return &singletons[(device >= 0 && device < 8) ? device : 0];
}

// Selection by name without touching the reference: simdjson resolves SIMDJSON_FORCE_IMPLEMENTATION against its own
// static list (src/implementation.cpp L211-242, L303), which an out-of-tree implementation cannot join.  When this
// library is loaded (linked or LD_PRELOADed) and the variable names "b200", it installs itself as the active
// implementation before the first use -- simdjson then never consults the list
// (get_active_implementation(), src/implementation.cpp L321-332).  SJB200_DEVICE picks the GPU (default 0).
namespace {
__attribute__((constructor)) void activate_if_forced() {
  const char *forced = std::getenv("SIMDJSON_FORCE_IMPLEMENTATION");
  if (forced == nullptr || std::strcmp(forced, "b200") != 0) return;
  const char *dev = std::getenv("SJB200_DEVICE");
  simdjson::get_active_implementation() = get_implementation(dev ? std::atoi(dev) : 0);
}
}  // namespace

// ---------------------------------------------------------------- dom_parser_implementation
dom_parser_implementation::~dom_parser_implementation() {
  if (ctx_ && pinned_) sjb200_unpin_host_memory(ctx_, pinned_);
  if (ctx_) sjb200_destroy(ctx_);
}

error_code dom_parser_implementation::ensure_context(size_t capacity) noexcept {
  if (!ctx_) return to_error(sjb200_create(device_, capacity, &ctx_));
  return to_error(sjb200_set_capacity(ctx_, capacity));
}

error_code dom_parser_implementation::set_capacity(size_t capacity) noexcept {
  // same contract as generic/dom_parser_implementation.h L66-82
  if (capacity > SIMDJSON_MAXSIZE_BYTES) return CAPACITY;
  const size_t words = SIMDJSON_ROUNDUP_N(capacity, 64) + 9;
  if (ctx_ && pinned_) { sjb200_unpin_host_memory(ctx_, pinned_); pinned_ = nullptr; }
  structural_indexes.reset(new (std::nothrow) uint32_t[words]);
  if (!structural_indexes) { _capacity = 0; return MEMALLOC; }
  structural_indexes[0] = 0;
  n_structural_indexes = 0;
  if (auto err = ensure_context(capacity)) { _capacity = 0; return err; }
  // the array must stay a plain new[] block (callers own it through unique_ptr<uint32_t[]>); page-lock it in place so
  // the index copy-back runs at PCIe speed (best effort: a failure only costs bandwidth)
  if (sjb200_pin_host_memory(ctx_, structural_indexes.get(), words * sizeof(uint32_t)) == SJB200_SUCCESS) pinned_ = structural_indexes.get();
  _capacity = capacity;
  return SUCCESS;
}

error_code dom_parser_implementation::set_max_depth(size_t max_depth) noexcept {
  if (!inner_) {
    // capacity 0: the inner parser never runs stage 1 and borrows our index array for stage 2
    if (auto err = simdjson::builtin_implementation()->create_dom_parser_implementation(0, max_depth, inner_)) return err;
  } else if (auto err = inner_->set_max_depth(max_depth)) {
    return err;
  }
  _max_depth = max_depth;
  return SUCCESS;
}

error_code dom_parser_implementation::stage1(const uint8_t *buf, size_t len, stage1_mode mode) noexcept {
  buf_ = buf;
  len_ = len;  // the reference keeps the untrimmed length here too (src/icelake.cpp L179-181)
  if (!ctx_) return UNINITIALIZED;
  gpu_calls_++;
  total_gpu_calls++;
  const int rc = sjb200_stage1(ctx_, buf, len, int(mode), structural_indexes.get(), &n_structural_indexes);
  // next_structural_index = 0 is stored together with the sentinels (json_structural_indexer.h L284-287),
  // i.e. on every path that got past the early returns
  bool early = (len > _capacity) || (len == 0) || rc == UNESCAPED_CHARS || rc == UNEXPECTED_ERROR || rc == MEMALLOC ||
               (rc == UNCLOSED_STRING && mode == stage1_mode::regular);
  if (!early && rc == UTF8_ERROR && mode != stage1_mode::regular) {
    // trim_partial_utf8 emptied the window (L198-204)
    size_t t = len;
    if (buf[len - 1] >= 0xC0) t = len - 1;
    else if (len >= 2 && buf[len - 2] >= 0xE0) t = len - 2;
    else if (len >= 3 && buf[len - 3] >= 0xF0) t = len - 3;
    early = (t == 0);
  }
  if (!early) next_structural_index = 0;
  return to_error(rc);
}

template <class F>
error_code dom_parser_implementation::with_inner(F &&f) noexcept {
  if (!inner_) return UNINITIALIZED;
  auto *cpu = static_cast<builtin_parser *>(inner_.get());
  cpu->buf = buf_;
  cpu->len = len_;
  cpu->_number_as_string = _number_as_string;  // dom::parser pokes these on the outer object (dom/parser-inl.h L136, L157-160)
  cpu->_unpadded = _unpadded;
  std::swap(cpu->structural_indexes, structural_indexes);
  cpu->n_structural_indexes = n_structural_indexes;
  cpu->next_structural_index = next_structural_index;
  const error_code err = f(*cpu);
  next_structural_index = cpu->next_structural_index;
  std::swap(cpu->structural_indexes, structural_indexes);
  return err;
}

error_code dom_parser_implementation::stage2(dom::document &doc) noexcept {
  return with_inner([&](builtin_parser &cpu) { return cpu.stage2(doc); });
}

error_code dom_parser_implementation::stage2_next(dom::document &doc) noexcept {
  return with_inner([&](builtin_parser &cpu) { return cpu.stage2_next(doc); });
}

error_code dom_parser_implementation::parse(const uint8_t *buf, size_t len, dom::document &doc) noexcept {
  if (auto err = stage1(buf, len, stage1_mode::regular)) return err;
  return stage2(doc);
}

uint8_t *dom_parser_implementation::parse_string(const uint8_t *src, uint8_t *dst, bool allow_replacement) const noexcept {
  return inner_ ? inner_->parse_string(src, dst, allow_replacement) : nullptr;
}

uint8_t *dom_parser_implementation::parse_wobbly_string(const uint8_t *src, uint8_t *dst) const noexcept {
  return inner_ ? inner_->parse_wobbly_string(src, dst) : nullptr;
}

}  // namespace b200
}  // namespace simdjson
