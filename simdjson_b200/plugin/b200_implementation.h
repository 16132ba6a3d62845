// b200_implementation.h -- the "b200" back-end for an UNMODIFIED simdjson.
//
// Two subclasses of simdjson's own plug-in classes (compiled against the reference's headers):
//
//   simdjson::b200::implementation             : simdjson::implementation
//        (include/simdjson/implementation.h L45-160)
//   simdjson::b200::dom_parser_implementation  : simdjson::internal::dom_parser_implementation
//        (include/simdjson/internal/dom_parser_implementation.h L48-242)
//
// stage1 / minify / validate_utf8 go to the GPU through the C ABI (include/sjb200.h); there is no CPU
// fallback for them.  Stage 2 (tape building) is out of scope for this path (SURVEY.md section 8, row 7)
// and is delegated to an inner parser of simdjson's built-in CPU implementation, which walks the
// index array the GPU produced.
//
// Install (doc/implementation-selection.md L93-110):
//     simdjson::get_active_implementation() = simdjson::b200::get_implementation();
// after which dom::parser::parse / parse_many, ondemand::parser::iterate, simdjson::minify and
// simdjson::validate_utf8 run their stage 1 on the H100.
#ifndef SIMDJSON_B200_IMPLEMENTATION_H
#define SIMDJSON_B200_IMPLEMENTATION_H

#include "simdjson.h"

extern "C" {
#include "sjb200.h"
}

namespace simdjson {
namespace b200 {

class implementation final : public simdjson::implementation {
 public:
  explicit implementation(int device = 0)
      : simdjson::implementation("b200", "NVIDIA H100 (sm_90a) stage 1", /*required_instruction_sets=*/0), device_(device) {}
  simdjson_warn_unused error_code create_dom_parser_implementation(size_t capacity, size_t max_depth,
                                                                   std::unique_ptr<internal::dom_parser_implementation> &dst) const noexcept final;
  simdjson_warn_unused error_code minify(const uint8_t *buf, size_t len, uint8_t *dst, size_t &dst_len) const noexcept final;
  simdjson_warn_unused bool validate_utf8(const char *buf, size_t len) const noexcept final;
  int device() const noexcept { return device_; }

 private:
  int device_;
};

class dom_parser_implementation final : public internal::dom_parser_implementation {
 public:
  explicit dom_parser_implementation(int device) noexcept : device_(device) {}
  ~dom_parser_implementation() override;
  dom_parser_implementation(const dom_parser_implementation &) = delete;
  dom_parser_implementation &operator=(const dom_parser_implementation &) = delete;

  simdjson_warn_unused error_code parse(const uint8_t *buf, size_t len, dom::document &doc) noexcept final;
  simdjson_warn_unused error_code stage1(const uint8_t *buf, size_t len, stage1_mode mode) noexcept final;
  simdjson_warn_unused error_code stage2(dom::document &doc) noexcept final;
  simdjson_warn_unused error_code stage2_next(dom::document &doc) noexcept final;
  simdjson_warn_unused uint8_t *parse_string(const uint8_t *src, uint8_t *dst, bool allow_replacement) const noexcept final;
  simdjson_warn_unused uint8_t *parse_wobbly_string(const uint8_t *src, uint8_t *dst) const noexcept final;
  error_code set_capacity(size_t capacity) noexcept final;
  error_code set_max_depth(size_t max_depth) noexcept final;

  // number of stage-1 calls this parser sent to the GPU (tests use it to prove the path taken)
  uint64_t gpu_stage1_calls() const noexcept { return gpu_calls_; }

 private:
  template <class F>
  error_code with_inner(F &&f) noexcept;  // lend the index array to the inner CPU parser around a stage-2 call
  error_code ensure_context(size_t capacity) noexcept;

  int device_;
  sjb200_ctx *ctx_{nullptr};
  std::unique_ptr<internal::dom_parser_implementation> inner_{};  // built-in CPU implementation: stage 2 only
  const uint8_t *buf_{nullptr};
  size_t len_{0};
  uint64_t gpu_calls_{0};
  void *pinned_{nullptr};  // the index array while it is page-locked
};

// the singleton to assign to simdjson::get_active_implementation()
const implementation *get_implementation(int device = 0) noexcept;

// stage-1 calls sent to the GPU by every parser of this process so far (the On-Demand parser keeps its
// implementation private, and a threaded document_stream swaps two parsers: tests count through this)
uint64_t gpu_stage1_calls_total() noexcept;

}  // namespace b200
}  // namespace simdjson

#endif
