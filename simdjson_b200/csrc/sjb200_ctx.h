// sjb200_ctx.h -- the context behind the C ABI (include/sjb200.h) and the host helpers its two translation units share:
// sjb200_capi.cu (lifetime, options, single-GPU calls, host-pointer pipeline) and sjb200_comm.cu (sharded passes).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/sjb200.h"
#include "sjb200_docs.h"
#include "sjb200_params.h"
#include "sjb200_tape.h"

namespace sjb200 {

class CopyPool;  // sjb200_hostpipe.h

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

constexpr int kCarrySlots = 1024;
constexpr int kTmapCacheEntries = 64;

struct TmapCacheEntry {
  const uint8_t *base = nullptr;
  uint64_t rows = 0;
  CUtensorMap map;
};
constexpr size_t kMaxBytes = 0xFFFFFFFFull;  // SIMDJSON_MAXSIZE_BYTES (include/simdjson/base.h L23)

struct PendingCall {
  int kind = -1;
  int mode = 0;
  int early_error = -1;  // >= 0: the call already failed / finished before any launch
  size_t len = 0;        // (trimmed) length scanned
  const uint8_t *d_buf = nullptr;
  uint32_t *d_idx = nullptr;
  uint8_t *d_dst = nullptr;
  cudaStream_t stream = nullptr;
  int carry_slot = 0;    // h_carry/d_carry slot holding the final carry
};

}  // namespace sjb200

struct sjb200_ctx {
  int device = 0;
  int sm_count = 0;
  size_t capacity = 0;
  cudaStream_t stream = nullptr;      // compute
  cudaStream_t copy_stream = nullptr; // H2D of the chunked host path
  cudaStream_t out_stream = nullptr;  // D2H of finished chunks' output
  std::vector<cudaEvent_t> chunk_events;
  // scratch
  uint8_t *d_in = nullptr;    size_t d_in_bytes = 0;
  uint32_t *d_idx = nullptr;  size_t d_idx_words = 0;
  uint8_t *d_out = nullptr;   size_t d_out_bytes = 0;
  sjb200::Carry *d_carry = nullptr;   // [kCarrySlots] one per chunk boundary of the chunked host pipeline
  // [0] the launch's flags, [1 + slot] the flags of the document whose result goes to carry slot `slot`, [1 + kCarrySlots]
  // the flags of a launch of parity 1 (launch_flags)
  uint32_t *d_flags = nullptr;
  uint32_t *d_ticket = nullptr;  // [parity][4]
  unsigned long long *d_count_desc = nullptr;  // [parity][desc_tiles]
  size_t desc_tiles = 0;
  unsigned long long *d_stamps = nullptr; size_t stamps_words = 0; size_t stamps_used = 0;  // option launch_stamps: [launch][2]
  sjb200::StreamFinish *d_sfin = nullptr;  // [kCarrySlots] results of the device-side streaming epilogue
  uint32_t *d_doc_scratch = nullptr; size_t doc_scratch_words = 0; uint32_t *d_ndocs = nullptr;
  uint8_t *d_tok_scratch = nullptr; size_t tok_scratch_bytes = 0; sjb200::TokenTotals *d_tok_tot = nullptr;  // stage-2-lite (sjb200_tape.cu)
  // JSON Pointer lookup (sjb200_pointer.cu): the compiled pointers, pinned and on the device (ptr_blob_bytes each), scratch
  uint8_t *h_ptr_blob = nullptr; uint8_t *d_ptr_blob = nullptr; size_t ptr_blob_bytes = 0;
  uint32_t *d_ptr_scratch = nullptr; size_t ptr_scratch_words = 0;
  uint32_t *d_gram_scratch = nullptr; size_t gram_scratch_words = 0;  // stage-2 grammar (sjb200_grammar.cu)
  uint64_t *d_col_scratch = nullptr; size_t col_scratch_words = 0;     // typed columns (sjb200_column.cu)
  int grid_u = 0;
  // pinned host mirrors
  sjb200::Carry *h_carry = nullptr;     // [kCarrySlots]
  uint32_t *h_flags = nullptr;
  uint8_t *h_small = nullptr;   // 64 B scratch
  sjb200::StreamFinish *h_sfin = nullptr;  // pinned mirror
  // batch: the last 3 bytes of every document.  Host and device blocks of tails_bytes each, laid out alike: [group]
  // pointers, [group] lengths, then 4 bytes per document coming back
  uint8_t *h_tails = nullptr; uint8_t *d_tails = nullptr; size_t tails_bytes = 0;
  uint32_t epoch = 0;
  int grid4 = 0;
  long opt_tok_stage = 1;
  long opt_use_tma = 1, opt_grid = 0, opt_chunk_bytes = 4 << 20, opt_time_kernel = 0;
  cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr;  // around the last scan kernel when opt_time_kernel is set
  bool ev_valid = false;
  std::vector<cudaEvent_t> ev_pool;              // [2i], [2i+1] around launch i since the last kernel_ms_mean query
  std::vector<uint32_t> ev_docs;                 // [i] documents launch i scanned
  size_t ev_used = 0;
  uint32_t ev_last_docs = 1;                     // ... the launch around ev_k0 / ev_k1
  // multi-document stage-1 launches: per group a DocEntry table and the documents' tensor maps, encoded for a whole
  // batch round into pinned memory, copied group by group ahead of the launches
  uint8_t *h_doctab = nullptr; uint8_t *d_doctab = nullptr; size_t doctab_bytes = 0;
  long opt_debug_timeline = 0;
  long opt_pdl = 1, opt_launch_stamps = 0;
  unsigned long long *d_debug = nullptr; size_t debug_words = 0; uint32_t debug_last_tiles = 0;
  unsigned long long launches = 0;               // kernels of ours launched by this context
  sjb200::PFN_encodeTiled encode = nullptr;
  sjb200::TmapCacheEntry tmap_cache[sjb200::kTmapCacheEntries];  // make_tensor_map
  // host-pointer pipeline: ring of page-locked staging slots filled by copy threads (sjb200_hostpipe.h)
  uint8_t *h_ring = nullptr; size_t ring_slot_bytes = 0; int ring_slots = 0;
  std::vector<cudaEvent_t> ring_events;
  sjb200::CopyPool *pool = nullptr;
  long opt_force_grid = 0;
  long opt_host_skip_scan = 0;  // tuning: the host-pointer pipeline copies only (no scan launches; results are meaningless)
  long opt_copy_threads = 4;        // 0: no staging (cudaMemcpyAsync straight from the caller's memory)
  long opt_ring_slots = 8;
  long opt_first_chunk_bytes = 512 << 10;  // first chunk of the host-pointer pipeline; the following ones double up to chunk_bytes
  long opt_stage_min_bytes = 1 << 20;  // smaller inputs go straight through the driver
  long opt_zero_copy_out = 1;       // stage 1 stores indexes straight into a page-locked, mapped caller array
  unsigned long long xchg_polls = 0, xchg_second_rounds = 0;  // sharded passes: window polls / passes that needed the second round
  double xchg_wait_ms = 0, xchg_evsync_ms = 0, xchg_enqueue_ms = 0;  // ... host time polling the window / waiting for the own scan / inside enqueue
  double t_wait_ms = 0, t_issue_ms = 0, t_sync_ms = 0;  // last host-pointer call: waiting for staged chunks / inside CUDA calls / final synchronise
  int last_input_path = 0, last_output_path = 0;  // stats: 0 driver copy, 1 staged ring, 2 caller memory is page-locked; 0 copy engine, 1 kernel stores
  sjb200::PendingCall pending;
  std::string last_error;
};

namespace sjb200 {

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

inline bool ok(sjb200_ctx *c, cudaError_t e, const char *what) {
  if (e == cudaSuccess) return true;
  c->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  (void)cudaGetLastError();
  return false;
}

template <typename T>
bool dev_alloc(sjb200_ctx *c, T **p, size_t count, const char *what) {
  void *q = nullptr;
  if (!ok(c, cudaMalloc(&q, count * sizeof(T)), what)) return false;
  *p = static_cast<T *>(q);
  return true;
}

// Grow-only device scratch of `*have` elements: when that is less than `need`, the old buffer is freed and `need` elements
// are allocated.  On a failure *p is null and *have 0.
template <typename T>
bool grow(sjb200_ctx *c, T **p, size_t *have, size_t need, const char *what) {
  if (*have >= need) return true;
  cudaFree(*p);
  *p = nullptr;
  *have = 0;
  if (!dev_alloc(c, p, need, what)) return false;
  *have = need;
  return true;
}

// the caller's stream, or the context's when it passes none
inline cudaStream_t stream_of(const sjb200_ctx *c, void *stream) { return stream ? static_cast<cudaStream_t>(stream) : c->stream; }

// ---- scan helpers (sjb200_capi.cu)
// scan4's look-back descriptors for a launch over `len` bytes (false: MEMALLOC)
bool ensure_desc(sjb200_ctx *c, size_t len);
// Enqueue the scan of the whole of (d_buf, len): kIndex into d_idx (sentinels: also the three words behind the last
// structural), kMinify into d_dst, kUtf8 neither.  carry_in null: the document starts here (zero state, zero count).
// The result goes to carry_out, and to carry_host too when given; xchg: a sharded launch's record (null: none).
// timed: inside the events of option time_kernel.
bool scan_document(sjb200_ctx *c, int kind, const uint8_t *d_buf, size_t len, uint32_t *d_idx, uint8_t *d_dst, bool sentinels, const Carry *carry_in,
                   Carry *carry_out, Carry *carry_host, const Xchg *xchg, cudaStream_t stream, bool timed);
// one small copy brings back everything a launch into carry slot 1 reports: {count, state, transducer, flags}
bool fetch_result(sjb200_ctx *c, cudaStream_t s);
// the partial-UTF-8 trim of a device buffer's end (json_structural_indexer.h L198-204); its last bytes come back first
bool trim_device_tail(sjb200_ctx *c, const uint8_t *d_buf, size_t *len, cudaStream_t s);

}  // namespace sjb200
