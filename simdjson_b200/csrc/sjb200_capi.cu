// sjb200_capi.cu -- the C ABI (include/sjb200.h): contexts, copies, launches and the host epilogue.
// No torch, no CPU fallback: every scan runs in sjb200_kernels.cu or the call fails.
#include <cuda.h>
#include <cuda_runtime.h>
#include <ctype.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <new>
#include <string>
#include <vector>

#include "../../include/sjb200.h"
#include "sjb200_bits.cuh"
#include "sjb200_docs.h"
#include "sjb200_tape.h"
#include "sjb200_finish.h"
#include "sjb200_hostpipe.h"
#include "sjb200_kernels.cuh"

using namespace sjb200;

namespace {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

constexpr int kCarrySlots = 1024;
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

}  // namespace

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
  Carry *d_carry = nullptr;   // [kCarrySlots] one per chunk boundary of the chunked host pipeline
  uint32_t *d_flags = nullptr;
  uint32_t *d_ticket = nullptr;
  unsigned long long *d_count_desc = nullptr;
  size_t desc_tiles = 0;
  StreamFinish *d_sfin = nullptr;  // [kCarrySlots] results of the device-side streaming epilogue
  uint32_t *d_doc_scratch = nullptr; size_t doc_scratch_words = 0; uint32_t *d_ndocs = nullptr;
  void *d_tok_scratch = nullptr; size_t tok_scratch_bytes = 0; TokenTotals *d_tok_tot = nullptr;  // stage-2-lite (sjb200_tape.cu)
  uint32_t *d_park = nullptr; size_t d_park_words = 0;  // scan4 with emit warps: parked masks (a per-CTA ring, independent of the input size)
  int grid_u = 0;
  // pinned host mirrors
  Carry *h_carry = nullptr;     // [kCarrySlots]
  uint32_t *h_flags = nullptr;
  uint8_t *h_small = nullptr;   // 64 B scratch
  StreamFinish *h_sfin = nullptr;  // pinned mirror
  uint8_t *h_tails = nullptr; uint8_t *d_tails = nullptr; const uint8_t **d_tail_ptrs = nullptr; size_t tails_cap = 0;  // batch: last 3 bytes of every document
  uint32_t epoch = 0;
  int grid4 = 0;
  long opt_tok_stage = 1;
  long opt_use_tma = 1, opt_grid = 0, opt_chunk_bytes = 4 << 20, opt_time_kernel = 0;
  cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr;  // around the last scan kernel when opt_time_kernel is set
  bool ev_valid = false;
  std::vector<cudaEvent_t> ev_pool;              // [2i], [2i+1] around launch i since the last kernel_ms_mean query
  size_t ev_used = 0;
  long opt_debug_timeline = 0;
  unsigned long long *d_debug = nullptr; size_t debug_tiles = 0; uint32_t debug_last_tiles = 0;
  unsigned long long launches = 0;               // kernels of ours launched by this context
  unsigned long long ew_launches = 0;            // ... of which stage-1 launches on the emit-warp build
  PFN_encodeTiled encode = nullptr;
  // host-pointer pipeline: ring of page-locked staging slots filled by copy threads (sjb200_hostpipe.h)
  uint8_t *h_ring = nullptr; size_t ring_slot_bytes = 0; int ring_slots = 0;
  std::vector<cudaEvent_t> ring_events;
  CopyPool *pool = nullptr;
  long opt_force_grid = 0;
  long opt_ew_min_bytes = 0;  // stage-1 launches of at least this many bytes run the emit-warp build of the kernel (0: never, the
                              // default: on H100 that build was slower at every launch size from 256 MiB to 1 GiB)
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
  PendingCall pending;
  std::string last_error;
};

namespace {

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

bool ok(sjb200_ctx *c, cudaError_t e, const char *what) {
  if (e == cudaSuccess) return true;
  c->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  (void)cudaGetLastError();
  return false;
}

size_t index_words(size_t capacity) { return ((capacity + 63) / 64) * 64 + 9; }
uint32_t tiles_of(size_t len) { return uint32_t((len + kTileBytes - 1) / kTileBytes); }

template <typename T>
bool dev_alloc(sjb200_ctx *c, T **p, size_t count, const char *what) {
  void *q = nullptr;
  if (!ok(c, cudaMalloc(&q, count * sizeof(T)), what)) return false;
  *p = static_cast<T *>(q);
  return true;
}

void free_sized(sjb200_ctx *c) {
  cudaFree(c->d_in); c->d_in = nullptr; c->d_in_bytes = 0;
  cudaFree(c->d_idx); c->d_idx = nullptr; c->d_idx_words = 0;
  cudaFree(c->d_out); c->d_out = nullptr; c->d_out_bytes = 0;
  cudaFree(c->d_count_desc); c->d_count_desc = nullptr;
  c->desc_tiles = 0;
}

// look-back descriptors: sized for the capacity, zeroed once (epoch tags make them reusable)
bool ensure_desc(sjb200_ctx *c, size_t len) {
  const size_t need = std::max<size_t>(tiles_of(len), 1);
  if (need <= c->desc_tiles) return true;
  cudaFree(c->d_count_desc); c->d_count_desc = nullptr;
  c->desc_tiles = 0;
  const size_t n = std::max(need, size_t(tiles_of(c->capacity)) + 1);
  if (!dev_alloc(c, &c->d_count_desc, n, "cudaMalloc(count_desc)")) return false;
  if (!ok(c, cudaMemsetAsync(c->d_count_desc, 0, n * sizeof(unsigned long long), c->stream), "memset desc")) return false;
  if (!ok(c, cudaStreamSynchronize(c->stream), "sync")) return false;
  c->desc_tiles = n;
  c->epoch = 0;
  return true;
}

// The wipe at the wrap of the 18-bit tag is ordered on the LAUNCH stream (a context is used on one stream at a time,
// see sjb200.h): kernels queued earlier on it finish before the wipe, the next launch starts after it.
bool next_epoch(sjb200_ctx *c, cudaStream_t launch_stream, uint32_t *epoch) {
  c->epoch++;
  if (c->epoch >= (1u << 18)) {
    if (!ok(c, cudaMemsetAsync(c->d_count_desc, 0, c->desc_tiles * sizeof(unsigned long long), launch_stream), "memset desc")) return false;
    c->epoch = 1;
  }
  *epoch = c->epoch;
  return true;
}

bool make_tensor_map(sjb200_ctx *c, CUtensorMap *map, const uint8_t *d_buf, size_t len, bool *usable, int box_rows = kScan4BoxRows) {
  memset(map, 0, sizeof(*map));
  *usable = false;
  const uint64_t rows = len / 128;
  if (!c->opt_use_tma || c->encode == nullptr || rows == 0) return true;
  if ((reinterpret_cast<uintptr_t>(d_buf) & 15u) != 0) return true;  // TMA needs a 16-byte aligned base
  cuuint64_t dims[2] = {128, rows};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {128, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = c->encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t *>(d_buf), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    c->last_error = "cuTensorMapEncodeTiled failed (" + std::to_string(int(r)) + "); using plain loads";
    return true;
  }
  *usable = true;
  return true;
}

// stage 1 and minify run on the scan4 structure (sjb200_scan4.cuh), validate_utf8 on utf8v2 (sjb200_utf8.cuh)
bool use_scan4(const sjb200_ctx *, int kind) { return kind == kIndex || kind == kMinify; }
// the one tensor map the kernel selected for `kind` reads through (scan4: 4 KiB boxes; the tile-synchronous kernels: 32 KiB)
bool map_for(sjb200_ctx *c, int kind, CUtensorMap *map, const uint8_t *d_buf, size_t len, bool *usable) {
  (void)kind;  // every kernel reads 4 KiB boxes of 32 rows
  return make_tensor_map(c, map, d_buf, len, usable, kScan4BoxRows);
}
int grid_cap(sjb200_ctx *c, int kind) {
  (void)kind;
  if (c->grid4 == 0) c->grid4 = scan4_max_ctas_per_sm() * c->sm_count;
  return c->opt_grid > 0 ? int(c->opt_grid) : c->grid4;
}
int grid_for(sjb200_ctx *c, int kind, uint32_t nelements) {
  if (c->opt_force_grid > 0) return int(c->opt_force_grid);  // tuning: a full grid even for a tiny document (measures the fixed cost of a launch)
  return int(std::max<uint32_t>(1, std::min<uint32_t>(uint32_t(grid_cap(c, kind)), nelements)));
}

// where a sharded launch publishes its record (sjb200_comm)
struct XchgTarget {
  unsigned long long *peer[kMaxRanks];
  uint32_t nranks, rank, slot, seq;
};

// Enqueue the scan of document tiles [tile_begin, tile_begin+ntiles) of (d_buf,len).
bool enqueue_scan(sjb200_ctx *c, int kind, const CUtensorMap *map, bool tma, const uint8_t *d_buf, size_t len, uint32_t tile_begin,
                  uint32_t ntiles, bool has_last_tile, uint32_t prev_word, uint32_t *d_idx, uint8_t *d_dst, int carry_in_slot,
                  cudaStream_t stream, int carry_out_slot = -1, bool write_sentinels = false, Carry *external_out = nullptr,
                  Carry *host_out = nullptr, const XchgTarget *xchg = nullptr) {
  // carry_in_slot < 0: the launch starts a document (zero state, zero count)
  if (carry_out_slot < 0) carry_out_slot = (carry_in_slot < 0) ? 1 : (carry_in_slot ^ 1);
  ScanParams p;
  memset(&p, 0, sizeof(p));
  p.buf = d_buf;
  p.len = len;
  p.pos_base = 0;
  p.prev_word = prev_word;
  p.check_eof = has_last_tile ? 1u : 0u;
  p.use_tma = tma ? 1u : 0u;
  p.tile_begin = tile_begin;
  p.ntiles = ntiles;
  if (!next_epoch(c, stream, &p.epoch)) return false;
  p.idx_out = d_idx;
  p.dst = d_dst;
  p.carry_in = (carry_in_slot < 0) ? nullptr : c->d_carry + carry_in_slot;
  p.write_sentinels = write_sentinels ? 1u : 0u;
  p.carry_out = external_out ? external_out : c->d_carry + carry_out_slot;
  p.carry_out_host = use_scan4(c, kind) ? host_out : nullptr;
  p.flags = c->d_flags;
  p.count_desc = c->d_count_desc;
  p.ticket = c->d_ticket;
  if (xchg && use_scan4(c, kind)) {
    for (int r = 0; r < kMaxRanks; r++) p.xchg_peer[r] = xchg->peer[r];
    p.xchg_nranks = xchg->nranks; p.xchg_rank = xchg->rank; p.xchg_slot = xchg->slot; p.xchg_seq = xchg->seq;
  }
  p.debug = nullptr;
  if (c->opt_debug_timeline) {
    const uint32_t rows = std::max<uint32_t>(ntiles, 4096);  // (the trace build of scan4 writes 17 rows per CTA)
    if (c->debug_tiles < rows) {
      cudaFree(c->d_debug); c->d_debug = nullptr; c->debug_tiles = 0;
      if (dev_alloc(c, &c->d_debug, size_t(rows) * 8, "cudaMalloc(debug)")) c->debug_tiles = rows;
    }
    if (c->d_debug) { cudaMemsetAsync(c->d_debug, 0, size_t(rows) * 64, stream); p.debug = c->d_debug; c->debug_last_tiles = rows; }
  }
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (c->opt_time_kernel) {
    if (c->ev_used + 2 > c->ev_pool.size() && c->ev_pool.size() < 4096) {
      cudaEvent_t a, b;
      cudaEventCreate(&a); cudaEventCreate(&b);
      c->ev_pool.push_back(a); c->ev_pool.push_back(b);
    }
    if (c->ev_used + 2 <= c->ev_pool.size()) { e0 = c->ev_pool[c->ev_used]; e1 = c->ev_pool[c->ev_used + 1]; c->ev_used += 2; }
    if (e0) cudaEventRecord(e0, stream);
  }
  bool launched;
  if (use_scan4(c, kind)) {
    const uint32_t tpe = uint32_t(scan4_tiles_per_element());
    const uint32_t nelem = (ntiles + tpe - 1) / tpe;
    const int grid = grid_for(c, kind, nelem);
    const bool ew = kind == kIndex && c->opt_ew_min_bytes > 0 && uint64_t(ntiles) * kTileBytes >= uint64_t(c->opt_ew_min_bytes);
    if (ew || scan4_parks_in_global()) {  // emit warps: the parked masks wait in an L2-resident ring of the context
      const size_t need = std::max(ew ? scan4_ew_park_words(grid_cap(c, kind)) : 0, scan4_parks_in_global() ? scan4_park_words(grid_cap(c, kind)) : 0);
      if (c->d_park_words < need) {
        cudaStreamSynchronize(c->stream);
        cudaFree(c->d_park); c->d_park = nullptr; c->d_park_words = 0;
        if (!dev_alloc(c, &c->d_park, need, "cudaMalloc(park)")) return false;
        c->d_park_words = need;
      }
      p.park = c->d_park;
    }
    launched = ew ? ok(c, launch_scan4_ew(map, p, grid, stream), "launch scan4 (emit warps)") : ok(c, launch_scan4(map, p, grid, kind == kMinify ? 2 : 0, stream), "launch scan4");
    c->ew_launches += (launched && ew) ? 1 : 0;
  } else {
    if (c->grid_u == 0) c->grid_u = utf8v2_max_ctas_per_sm() * c->sm_count;
    const uint64_t nblocks = (uint64_t(ntiles) * kTileBytes + 4095) / 4096;
    const uint64_t want = (nblocks + uint64_t(utf8v2_warps_per_cta()) - 1) / uint64_t(utf8v2_warps_per_cta());
    const int grid = c->opt_force_grid > 0 ? int(c->opt_force_grid) : int(std::max<uint64_t>(1, std::min<uint64_t>(uint64_t(c->opt_grid > 0 ? c->opt_grid : c->grid_u), want)));
    p.carry_out_host = host_out;
    launched = ok(c, launch_utf8v2(map, p, grid, stream), "launch utf8v2");
  }
  if (e1) { cudaEventRecord(e1, stream); c->ev_k0 = e0; c->ev_k1 = e1; c->ev_valid = launched; }
  c->launches += launched ? 1 : 0;
  return launched;
}

// (the streaming modes' walk over the tail of a device-resident index array lives on the device: sjb200_docs.cu)
class NullIndexWriter final : public IndexWriter {  // regular mode behind a device-resident scan: the kernel stored the sentinels already
 public:
  bool set3(uint32_t, uint32_t, uint32_t, uint32_t) override { return false; }
  bool final_fixup(uint32_t, uint32_t) override { return false; }
};
class NullReader final : public StructuralReader {
 public:
  uint32_t position(uint32_t) override { return 0; }
  uint8_t character(uint32_t) override { return 0; }
};

bool is_filter_mode(int mode) { return mode >= SJB200_JSON_SEQUENCE_PARTIAL; }

// one small copy brings back everything a launch reports: {count, state, transducer, flags} of slot 1
bool fetch_result(sjb200_ctx *c, cudaStream_t s) {
  return ok(c, cudaMemcpyAsync(c->h_carry + 1, c->d_carry + 1, sizeof(Carry), cudaMemcpyDeviceToHost, s), "D2H result");
}

}  // namespace

// =============================================================================== lifetime
extern "C" size_t sjb200_index_words(size_t capacity) { return index_words(capacity); }

extern "C" int sjb200_create(int device, size_t capacity, sjb200_ctx **out) {
  if (!out) return SJB200_UNEXPECTED_ERROR;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
    (void)cudaGetLastError();
    return SJB200_UNSUPPORTED_ARCHITECTURE;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
    (void)cudaGetLastError();
    return SJB200_UNSUPPORTED_ARCHITECTURE;  // the kernel image is sm_90a only
  }
  sjb200_ctx *c = new (std::nothrow) sjb200_ctx();
  if (!c) return SJB200_MEMALLOC;
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  DeviceGuard g(device);
  bool good = ok(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking), "stream") &&
              ok(c, cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking), "stream") &&
              ok(c, cudaStreamCreateWithFlags(&c->out_stream, cudaStreamNonBlocking), "stream") &&
              dev_alloc(c, &c->d_carry, kCarrySlots, "cudaMalloc(carry)") && dev_alloc(c, &c->d_flags, 1, "cudaMalloc(flags)") &&
              dev_alloc(c, &c->d_ticket, 4, "cudaMalloc(ticket)") &&
              ok(c, cudaMemset(c->d_ticket, 0, 4 * sizeof(uint32_t)), "memset ticket") &&
              ok(c, cudaMemset(c->d_flags, 0, sizeof(uint32_t)), "memset flags");
  void *hp = nullptr;
  good = good && ok(c, cudaMallocHost(&hp, kCarrySlots * sizeof(Carry)), "cudaMallocHost");
  c->h_carry = static_cast<Carry *>(hp);
  good = good && ok(c, cudaMallocHost(&hp, sizeof(uint32_t)), "cudaMallocHost");
  c->h_flags = static_cast<uint32_t *>(hp);
  good = good && ok(c, cudaMallocHost(&hp, 64), "cudaMallocHost");
  c->h_small = static_cast<uint8_t *>(hp);
  good = good && ok(c, cudaMallocHost(&hp, kCarrySlots * sizeof(StreamFinish)), "cudaMallocHost");
  c->h_sfin = static_cast<StreamFinish *>(hp);
  good = good && dev_alloc(c, &c->d_sfin, kCarrySlots, "cudaMalloc(stream finish)") && dev_alloc(c, &c->d_ndocs, 1, "cudaMalloc(ndocs)");
  if (good) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      c->encode = reinterpret_cast<PFN_encodeTiled>(fn);
    else
      (void)cudaGetLastError();
  }
  if (!good) {
    sjb200_destroy(c);
    return SJB200_MEMALLOC;
  }
  // tuning knobs of the host-pointer pipeline for callers that cannot reach sjb200_set_option (the C++ plug-in owns its contexts)
  for (const char *key : {"copy_threads", "ring_slots", "chunk_bytes", "first_chunk_bytes", "stage_min_bytes", "zero_copy_out"}) {
    std::string env = std::string("SJB200_") + key;
    for (auto &ch : env) ch = char(toupper((unsigned char)ch));
    if (const char *v = getenv(env.c_str())) sjb200_set_option(c, key, atol(v));
  }
  int rc = sjb200_set_capacity(c, capacity);
  if (rc != SJB200_SUCCESS) {
    sjb200_destroy(c);
    return rc;
  }
  *out = c;
  return SJB200_SUCCESS;
}

extern "C" void sjb200_destroy(sjb200_ctx *c) {
  if (!c) return;
  DeviceGuard g(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  free_sized(c);
  cudaFree(c->d_carry); cudaFree(c->d_flags); cudaFree(c->d_ticket); cudaFree(c->d_sfin); cudaFree(c->d_doc_scratch); cudaFree(c->d_ndocs); cudaFree(c->d_tok_scratch); cudaFree(c->d_tok_tot); cudaFree(c->d_tails); cudaFree(c->d_tail_ptrs); cudaFree(c->d_debug); cudaFree(c->d_park);
  if (c->h_carry) cudaFreeHost(c->h_carry);
  if (c->h_flags) cudaFreeHost(c->h_flags);
  if (c->h_small) cudaFreeHost(c->h_small);
  if (c->h_sfin) cudaFreeHost(c->h_sfin);
  if (c->h_tails) cudaFreeHost(c->h_tails);
  delete c->pool; c->pool = nullptr;
  if (c->h_ring) cudaFreeHost(c->h_ring);
  for (auto e : c->ring_events) cudaEventDestroy(e);
  for (auto e : c->ev_pool) cudaEventDestroy(e);
  for (auto e : c->chunk_events) cudaEventDestroy(e);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->out_stream) cudaStreamDestroy(c->out_stream);
  delete c;
}

extern "C" int sjb200_set_capacity(sjb200_ctx *c, size_t capacity) {
  if (!c) return SJB200_UNEXPECTED_ERROR;
  if (capacity > kMaxBytes) return SJB200_CAPACITY;  // generic/dom_parser_implementation.h L67
  DeviceGuard g(c->device);
  if (capacity != c->capacity) {
    cudaStreamSynchronize(c->stream);
    free_sized(c);  // host-path staging buffers are re-created lazily at the new size
  }
  c->capacity = capacity;
  if (!ensure_desc(c, capacity)) return SJB200_MEMALLOC;
  return SJB200_SUCCESS;
}

extern "C" size_t sjb200_capacity(const sjb200_ctx *c) { return c ? c->capacity : 0; }
extern "C" int sjb200_device(const sjb200_ctx *c) { return c ? c->device : -1; }
extern "C" const char *sjb200_last_cuda_error(const sjb200_ctx *c) { return c ? c->last_error.c_str() : ""; }

// tuning aid: copy the per-tile timeline of the last launch (8 x uint64 per tile) to host memory; returns tiles copied
extern "C" long sjb200_get_debug_timeline(sjb200_ctx *c, unsigned long long *out, size_t max_tiles) {
  if (!c || !c->d_debug || !out) return 0;
  DeviceGuard g(c->device);
  const size_t n = std::min<size_t>(max_tiles, c->debug_last_tiles);
  cudaDeviceSynchronize();
  if (cudaMemcpy(out, c->d_debug, n * 64, cudaMemcpyDeviceToHost) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  return long(n);
}

extern "C" int sjb200_pin_host_memory(sjb200_ctx *c, void *ptr, size_t bytes) {
  if (!c || !ptr || bytes == 0) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  return ok(c, cudaHostRegister(ptr, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped), "cudaHostRegister") ? SJB200_SUCCESS : SJB200_MEMALLOC;
}
extern "C" int sjb200_unpin_host_memory(sjb200_ctx *c, void *ptr) {
  if (!c || !ptr) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  return ok(c, cudaHostUnregister(ptr), "cudaHostUnregister") ? SJB200_SUCCESS : SJB200_UNEXPECTED_ERROR;
}

extern "C" double sjb200_get_stat(sjb200_ctx *c, const char *key) {
  if (!c || !key) return -1.0;
  if (!strcmp(key, "kernel_ms")) {  // duration of the last scan kernel (needs option time_kernel=1 and a finished call)
    if (!c->ev_valid) return -1.0;
    DeviceGuard g(c->device);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev_k0, c->ev_k1) != cudaSuccess) { (void)cudaGetLastError(); return -1.0; }
    return double(ms);
  }
  if (!strcmp(key, "kernel_ms_mean")) {  // mean duration of the scan kernels launched since the previous query
    DeviceGuard g(c->device);
    double sum = 0;
    size_t n = 0;
    for (size_t i = 0; i + 1 < c->ev_used; i += 2) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, c->ev_pool[i], c->ev_pool[i + 1]) == cudaSuccess) { sum += ms; n++; } else (void)cudaGetLastError();
    }
    c->ev_used = 0;
    c->ev_valid = false;
    return n ? sum / double(n) : -1.0;
  }
  if (!strcmp(key, "launches")) return double(c->launches);
  if (!strcmp(key, "ew_launches")) return double(c->ew_launches);
  if (!strcmp(key, "grid_index")) return double(grid_for(c, kIndex, 0xFFFFFFFFu));
  if (!strcmp(key, "sm_count")) return double(c->sm_count);
  if (!strcmp(key, "host_wait_ms")) return c->t_wait_ms;
  if (!strcmp(key, "xchg_polls")) return double(c->xchg_polls);
  if (!strcmp(key, "xchg_second_rounds")) return double(c->xchg_second_rounds);
  if (!strcmp(key, "xchg_wait_ms")) return c->xchg_wait_ms;
  if (!strcmp(key, "xchg_evsync_ms")) return c->xchg_evsync_ms;
  if (!strcmp(key, "xchg_enqueue_ms")) return c->xchg_enqueue_ms;
  if (!strcmp(key, "host_issue_ms")) return c->t_issue_ms;
  if (!strcmp(key, "host_sync_ms")) return c->t_sync_ms;
  if (!strcmp(key, "input_path")) return double(c->last_input_path);
  if (!strcmp(key, "output_path")) return double(c->last_output_path);
  return -1.0;
}

extern "C" int sjb200_set_option(sjb200_ctx *c, const char *key, long value) {
  if (!c || !key) return SJB200_UNEXPECTED_ERROR;
  if (!strcmp(key, "use_tma")) c->opt_use_tma = value;
  else if (!strcmp(key, "grid")) c->opt_grid = value;
  else if (!strcmp(key, "tok_stage")) c->opt_tok_stage = value ? 1 : 0;
  else if (!strcmp(key, "time_kernel")) c->opt_time_kernel = value;
  else if (!strcmp(key, "debug_timeline")) c->opt_debug_timeline = value;
  else if (!strcmp(key, "chunk_bytes")) c->opt_chunk_bytes = std::max<long>(2 * kTileBytes, (value / (2 * kTileBytes)) * (2 * kTileBytes));
  else if (!strcmp(key, "force_grid")) c->opt_force_grid = value;
  else if (!strcmp(key, "ew_min_bytes")) c->opt_ew_min_bytes = value;
  else if (!strcmp(key, "host_skip_scan")) c->opt_host_skip_scan = value;
  else if (!strcmp(key, "copy_threads")) c->opt_copy_threads = std::max<long>(0, std::min<long>(value, 64));
  else if (!strcmp(key, "ring_slots")) c->opt_ring_slots = std::max<long>(2, std::min<long>(value, 64));
  else if (!strcmp(key, "stage_min_bytes")) c->opt_stage_min_bytes = std::max<long>(0, value);
  else if (!strcmp(key, "first_chunk_bytes")) c->opt_first_chunk_bytes = std::max<long>(2 * kTileBytes, (value / (2 * kTileBytes)) * (2 * kTileBytes));
  else if (!strcmp(key, "zero_copy_out")) c->opt_zero_copy_out = value;
  else return SJB200_UNEXPECTED_ERROR;
  return SJB200_SUCCESS;
}

// =============================================================================== device-resident
namespace {
// enqueue one device-resident stage-1 scan; its {count,state,flags} come back in h_carry[slot]
void stage1_enqueue_into(sjb200_ctx *c, PendingCall &pc, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, cudaStream_t s,
                         int slot, const uint8_t *tail3 = nullptr /* host copy of the last min(3, len) bytes, when the caller fetched it */) {
  pc = PendingCall();
  pc.kind = kIndex; pc.mode = mode; pc.d_buf = d_buf; pc.d_idx = d_idx; pc.stream = s; pc.len = len; pc.carry_slot = slot;
  if (mode < SJB200_REGULAR || mode > SJB200_COMMA_DELIMITED_FINAL) { pc.early_error = SJB200_UNEXPECTED_ERROR; return; }
  if (len > c->capacity) { pc.early_error = SJB200_CAPACITY; return; }   // json_structural_indexer.h L195
  if (len == 0) { pc.early_error = SJB200_EMPTY; return; }                // L197
  if (mode != SJB200_REGULAR) {                                           // L198-204
    const size_t k = std::min<size_t>(3, len);
    if (!tail3) {
      if (!ok(c, cudaMemcpyAsync(c->h_small, d_buf + len - k, k, cudaMemcpyDeviceToHost, s), "D2H tail") ||
          !ok(c, cudaStreamSynchronize(s), "sync"))
        { pc.early_error = SJB200_UNEXPECTED_ERROR; return; }
      tail3 = c->h_small;
    }
    len = trim_partial_utf8_tail(tail3, k, len);
    pc.len = len;
    if (len == 0) { pc.early_error = SJB200_UTF8_ERROR; return; }
  }
  if (!ensure_desc(c, len)) { pc.early_error = SJB200_MEMALLOC; return; }
  CUtensorMap map;
  bool tma = false;
  map_for(c, kIndex, &map, d_buf, len, &tma);
  // scan4 stores its result in the pinned host mirror itself; the older kernel needs the copy engine for it
  if (!enqueue_scan(c, kIndex, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, d_idx, nullptr, -1, s, slot, true, nullptr,
                    c->h_carry + slot) ||
      (!use_scan4(c, kIndex) &&
       !ok(c, cudaMemcpyAsync(c->h_carry + slot, c->d_carry + slot, sizeof(Carry), cudaMemcpyDeviceToHost, s), "D2H result")))
    { pc.early_error = SJB200_UNEXPECTED_ERROR; return; }
  // whitespace-separated streams: the rest of finish() (find_next_document_index, the final fix-up) runs on the device
  // right behind the scan -- no host round trip between the two (sjb200_docs.cu)
  if (mode == SJB200_STREAMING_PARTIAL || mode == SJB200_STREAMING_FINAL) {
    c->launches++;
    if (!ok(c, launch_stream_finish(d_buf, d_idx, c->d_carry + slot, uint32_t(len), mode, c->d_sfin + slot, c->h_sfin + slot, s), "stream finish"))
      pc.early_error = SJB200_UNEXPECTED_ERROR;
  }
}

// complete one enqueued scan (the stream has been synchronised by the caller)
int stage1_finish_from(sjb200_ctx *c, const PendingCall &pc, uint32_t *n_inout) {
  if (pc.early_error >= 0) return pc.early_error;
  if (pc.mode == SJB200_STREAMING_PARTIAL || pc.mode == SJB200_STREAMING_FINAL) {
    const StreamFinish &r = c->h_sfin[pc.carry_slot];  // written by stream_finish_kernel behind the scan
    if (r.n_written && n_inout) *n_inout = r.n;
    return r.err;
  }
  FinishInput in;
  in.mode = pc.mode; in.len = pc.len;
  in.count = c->h_carry[pc.carry_slot].count;
  in.state = c->h_carry[pc.carry_slot].state;
  in.flags = c->h_carry[pc.carry_slot].flags;
  in.sentinels_written = true;
  int rc;
  uint32_t n_local = n_inout ? *n_inout : 0;
  if (is_filter_mode(pc.mode)) {
    // RS / comma-delimited streams: the filters and the rest of finish() run on the device-resident array (sjb200_docs.cu);
    // only the error precedence that needs no data is decided here (json_structural_indexer.h L249-291)
    if (in.flags & kFlagInternal) return SJB200_UNEXPECTED_ERROR;
    if (in.flags & kFlagCtl) return SJB200_UNESCAPED_CHARS;
    uint32_t n = uint32_t(in.count);
    n_local = n;
    if (n == 0) { if (n_inout) *n_inout = 0; return SJB200_EMPTY; }
    const bool unclosed = (in.state >> 1) & 1u;
    const bool partial = (pc.mode == SJB200_JSON_SEQUENCE_PARTIAL || pc.mode == SJB200_COMMA_DELIMITED_PARTIAL);
    if (unclosed) {
      n--;
      if (partial) { n_local = n; if (n == 0) { if (n_inout) *n_inout = 0; return SJB200_CAPACITY; } }
    }
    const size_t need = filter_scratch_words(n);
    if (c->doc_scratch_words < need) {
      cudaFree(c->d_doc_scratch); c->d_doc_scratch = nullptr; c->doc_scratch_words = 0;
      if (!dev_alloc(c, &c->d_doc_scratch, need, "cudaMalloc(filter scratch)")) return SJB200_MEMALLOC;
      c->doc_scratch_words = need;
    }
    c->launches += 4;
    if (!ok(c, launch_stream_filter(pc.d_buf, uint32_t(pc.len), pc.d_idx, n, pc.mode, in.flags, c->d_doc_scratch, c->d_sfin + pc.carry_slot,
                                    c->h_sfin + pc.carry_slot, pc.stream), "stream filter") ||
        !ok(c, cudaStreamSynchronize(pc.stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    const StreamFinish &r = c->h_sfin[pc.carry_slot];
    if (n_inout) *n_inout = r.n;
    return r.err;
  } else {  // regular: error precedence only, nothing to read or write (the scan stored the sentinels)
    NullReader reader;
    NullIndexWriter writer;
    bool dirty = false;
    rc = finish_stage1(in, reader, writer, &n_local, nullptr, nullptr, &dirty);
  }
  if (n_inout) *n_inout = n_local;
  return rc;
}

}  // namespace

extern "C" int sjb200_stage1_dev_enqueue(sjb200_ctx *c, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, void *stream) {
  if (!c) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  stage1_enqueue_into(c, c->pending, d_buf, len, mode, d_idx, stream ? static_cast<cudaStream_t>(stream) : c->stream, 1);
  return SJB200_SUCCESS;
}

extern "C" int sjb200_stage1_dev_finish(sjb200_ctx *c, uint32_t *n_inout) {
  if (!c || c->pending.kind != kIndex) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  PendingCall pc = c->pending;
  c->pending.kind = -1;
  if (pc.early_error < 0 && !ok(c, cudaStreamSynchronize(pc.stream), "sync")) return SJB200_UNEXPECTED_ERROR;
  return stage1_finish_from(c, pc, n_inout);
}

// Many documents in one call (NDJSON rows, a corpus): every scan is queued back to back on the stream, the host
// waits once, then completes each document's finish() logic.  docs[i].error receives the error_code.
extern "C" int sjb200_stage1_dev_batch(sjb200_ctx *c, sjb200_doc *docs, int ndocs, int mode, void *stream) {
  if (!c || (!docs && ndocs > 0) || ndocs < 0) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  std::vector<PendingCall> calls;
  int done = 0;
  while (done < ndocs) {
    const int group = std::min(ndocs - done, kCarrySlots - 2);  // one result slot per document in flight
    calls.assign(size_t(group), PendingCall());
    const uint8_t *tails = nullptr;
    if (mode != SJB200_REGULAR) {
      // streaming modes look at every document's last three bytes before its scan (partial UTF-8 tail): fetch them for
      // the whole group with one launch and one copy instead of one synchronous copy per document
      if (c->tails_cap < size_t(group)) {
        if (c->h_tails) cudaFreeHost(c->h_tails);
        cudaFree(c->d_tails); cudaFree(c->d_tail_ptrs);
        c->h_tails = nullptr; c->d_tails = nullptr; c->d_tail_ptrs = nullptr; c->tails_cap = 0;
        void *hp = nullptr;
        // host block: [group] pointers, [group] lengths, then 4 bytes per document coming back
        if (!ok(c, cudaMallocHost(&hp, size_t(group) * 20), "cudaMallocHost(tails)") || !dev_alloc(c, &c->d_tails, size_t(group) * 4, "cudaMalloc(tails)") ||
            !dev_alloc(c, &c->d_tail_ptrs, size_t(group) * 2, "cudaMalloc(tail ptrs)"))
          return SJB200_MEMALLOC;
        c->h_tails = static_cast<uint8_t *>(hp);
        c->tails_cap = size_t(group);
      }
      const uint8_t **hptr = reinterpret_cast<const uint8_t **>(c->h_tails);
      uint64_t *hlen = reinterpret_cast<uint64_t *>(c->h_tails + size_t(group) * 8);
      uint8_t *hout = c->h_tails + size_t(group) * 16;
      for (int i = 0; i < group; i++) { hptr[i] = docs[done + i].d_buf; hlen[i] = (docs[done + i].len <= c->capacity) ? docs[done + i].len : 0; }
      const uint64_t *dlen = reinterpret_cast<const uint64_t *>(c->d_tail_ptrs + group);
      if (!ok(c, cudaMemcpyAsync(c->d_tail_ptrs, c->h_tails, size_t(group) * 16, cudaMemcpyHostToDevice, s), "H2D tail ptrs") ||
          !ok(c, launch_gather_tails(c->d_tail_ptrs, dlen, uint32_t(group), c->d_tails, s), "gather tails") ||
          !ok(c, cudaMemcpyAsync(hout, c->d_tails, size_t(group) * 4, cudaMemcpyDeviceToHost, s), "D2H tails") || !ok(c, cudaStreamSynchronize(s), "sync"))
        return SJB200_UNEXPECTED_ERROR;
      c->launches++;
      tails = hout;
    }
    for (int i = 0; i < group; i++) {
      sjb200_doc &d = docs[done + i];
      stage1_enqueue_into(c, calls[size_t(i)], d.d_buf, d.len, mode, d.d_idx, s, 1 + i, tails ? tails + 4 * size_t(i) : nullptr);
    }
    if (!ok(c, cudaStreamSynchronize(s), "sync")) return SJB200_UNEXPECTED_ERROR;
    for (int i = 0; i < group; i++) {
      sjb200_doc &d = docs[done + i];
      d.error = stage1_finish_from(c, calls[size_t(i)], &d.n_structural_indexes);
    }
    done += group;
  }
  return SJB200_SUCCESS;
}

// every place a document of a whitespace-separated stream starts (SURVEY.md 8(f) row 1): built on the device from a
// device-resident index array, in stream order
extern "C" int sjb200_document_table_dev(sjb200_ctx *c, const uint8_t *d_buf, const uint32_t *d_idx, uint32_t n, sjb200_doc_boundary *d_table,
                                         uint32_t capacity, uint32_t *ndocs_out, void *stream) {
  if (!c || !d_buf || !d_idx || !ndocs_out || (capacity && !d_table)) return SJB200_UNEXPECTED_ERROR;
  *ndocs_out = 0;
  if (n == 0) return SJB200_SUCCESS;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  const size_t need = doc_table_scratch_words(n);
  if (c->doc_scratch_words < need) {
    cudaFree(c->d_doc_scratch); c->d_doc_scratch = nullptr; c->doc_scratch_words = 0;
    if (!dev_alloc(c, &c->d_doc_scratch, need, "cudaMalloc(doc scratch)")) return SJB200_MEMALLOC;
    c->doc_scratch_words = need;
  }
  static_assert(sizeof(sjb200_doc_boundary) == sizeof(sjb200_doc_boundary_t), "layout");
  if (!ok(c, launch_doc_table(d_buf, d_idx, n, c->d_doc_scratch, reinterpret_cast<sjb200_doc_boundary_t *>(d_table), capacity, c->d_ndocs, s), "doc table") ||
      !ok(c, cudaMemcpyAsync(c->h_small, c->d_ndocs, sizeof(uint32_t), cudaMemcpyDeviceToHost, s), "D2H ndocs") || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += 3;
  memcpy(ndocs_out, c->h_small, sizeof(uint32_t));
  return SJB200_SUCCESS;
}

// stage-2-lite (SURVEY.md 8(f) row 4): type and payload of every token, the document's string buffer -- sjb200_tape.cu
extern "C" size_t sjb200_string_buf_capacity(size_t len) { return ((5 * (len / 3) + 64) + 63) / 64 * 64; }  // dom/document-inl.h L54

extern "C" int sjb200_tokens_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, const uint32_t *d_idx, uint32_t n, uint8_t *d_type, uint64_t *d_payload,
                                 uint8_t *d_strbuf, size_t strbuf_capacity, sjb200_tokens_result *out, void *stream) {
  if (!c || !out || (n && (!d_buf || !d_idx || !d_type || !d_payload)) || (strbuf_capacity && !d_strbuf)) return SJB200_UNEXPECTED_ERROR;
  out->error = SJB200_SUCCESS; out->first_error_index = 0xFFFFFFFFu; out->n_strings = 0; out->string_bytes = 0;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  const size_t need = tokens_scratch_bytes(n);
  if (c->tok_scratch_bytes < need) {
    cudaFree(c->d_tok_scratch); c->d_tok_scratch = nullptr; c->tok_scratch_bytes = 0;
    if (cudaMalloc(&c->d_tok_scratch, need) != cudaSuccess) { c->last_error = "cudaMalloc(token scratch)"; return SJB200_MEMALLOC; }
    c->tok_scratch_bytes = need;
  }
  if (!c->d_tok_tot && cudaMalloc(reinterpret_cast<void **>(&c->d_tok_tot), sizeof(TokenTotals)) != cudaSuccess) { c->last_error = "cudaMalloc(token totals)"; return SJB200_MEMALLOC; }
  static_assert(sizeof(TokenTotals) <= 64, "h_small");
  if (!ok(c, launch_tokens(d_buf, len, d_idx, n, d_type, d_payload, d_strbuf, strbuf_capacity, c->d_tok_scratch, c->d_tok_tot, int(c->opt_tok_stage), s), "tokens") ||
      !ok(c, cudaMemcpyAsync(c->h_small, c->d_tok_tot, sizeof(TokenTotals), cudaMemcpyDeviceToHost, s), "D2H token totals") || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += n ? 3 : 1;
  TokenTotals t;
  memcpy(&t, c->h_small, sizeof(t));
  out->n_strings = t.n_strings;
  out->string_bytes = t.string_bytes;
  if (t.first_error != ~0ull) {
    out->first_error_index = uint32_t(t.first_error >> 8);
    out->error = int(t.first_error & 0xFFull);
  } else if (t.string_bytes > strbuf_capacity) {
    out->error = SJB200_CAPACITY;
  }
  return out->error;
}

extern "C" int sjb200_stage1_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, uint32_t *n_inout,
                                 void *stream) {
  int rc = sjb200_stage1_dev_enqueue(c, d_buf, len, mode, d_idx, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_stage1_dev_finish(c, n_inout);
}

extern "C" int sjb200_minify_dev_enqueue(sjb200_ctx *c, const uint8_t *d_buf, size_t len, uint8_t *d_dst, void *stream) {
  if (!c) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  PendingCall &pc = c->pending;
  pc = PendingCall();
  pc.kind = kMinify; pc.d_buf = d_buf; pc.d_dst = d_dst; pc.stream = s; pc.len = len;
  if (len > kMaxBytes) { pc.early_error = SJB200_CAPACITY; return SJB200_SUCCESS; }
  if (len == 0) { pc.early_error = SJB200_SUCCESS; return SJB200_SUCCESS; }  // json_minifier.h: nothing to do, dst_len = 0
  if (!ensure_desc(c, len)) { pc.early_error = SJB200_MEMALLOC; return SJB200_SUCCESS; }
  CUtensorMap map;
  bool tma = false;
  map_for(c, kMinify, &map, d_buf, len, &tma);
  if (!enqueue_scan(c, kMinify, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, nullptr, d_dst, -1, s, 1) ||
      !fetch_result(c, s))
    pc.early_error = SJB200_UNEXPECTED_ERROR;
  pc.carry_slot = 1;
  return SJB200_SUCCESS;
}

extern "C" int sjb200_minify_dev_finish(sjb200_ctx *c, size_t *dst_len) {
  if (!c || c->pending.kind != kMinify) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  PendingCall pc = c->pending;
  c->pending.kind = -1;
  if (dst_len) *dst_len = 0;
  if (pc.early_error >= 0) return pc.early_error;
  if (!ok(c, cudaStreamSynchronize(pc.stream), "sync")) return SJB200_UNEXPECTED_ERROR;
  if (c->h_carry[pc.carry_slot].flags & kFlagInternal) return SJB200_UNEXPECTED_ERROR;
  if ((c->h_carry[pc.carry_slot].state >> 1) & 1u) return SJB200_UNCLOSED_STRING;  // json_minifier.h L42-47
  if (dst_len) *dst_len = size_t(c->h_carry[pc.carry_slot].count);
  return SJB200_SUCCESS;
}

extern "C" int sjb200_minify_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, uint8_t *d_dst, size_t *dst_len, void *stream) {
  int rc = sjb200_minify_dev_enqueue(c, d_buf, len, d_dst, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_minify_dev_finish(c, dst_len);
}

extern "C" int sjb200_validate_utf8_dev_enqueue(sjb200_ctx *c, const uint8_t *d_buf, size_t len, void *stream) {
  if (!c) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  PendingCall &pc = c->pending;
  pc = PendingCall();
  pc.kind = kUtf8; pc.d_buf = d_buf; pc.stream = s; pc.len = len;
  if (len == 0) { pc.early_error = SJB200_SUCCESS; return SJB200_SUCCESS; }  // utf8_validator.h L27-28: empty is valid
  if (len > kMaxBytes) { pc.early_error = SJB200_CAPACITY; return SJB200_SUCCESS; }
  CUtensorMap map;
  bool tma = false;
  map_for(c, kUtf8, &map, d_buf, len, &tma);
  if (!enqueue_scan(c, kUtf8, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, nullptr, nullptr, -1, s, 1) ||
      !fetch_result(c, s))
    pc.early_error = SJB200_UNEXPECTED_ERROR;
  return SJB200_SUCCESS;
}

// returns 1 valid, 0 invalid, negative = CUDA failure
extern "C" int sjb200_validate_utf8_dev_finish(sjb200_ctx *c) {
  if (!c || c->pending.kind != kUtf8) return -1;
  DeviceGuard g(c->device);
  PendingCall pc = c->pending;
  c->pending.kind = -1;
  if (pc.early_error == SJB200_SUCCESS) return 1;
  if (pc.early_error > 0) return -1;
  if (!ok(c, cudaStreamSynchronize(pc.stream), "sync")) return -1;
  if (c->h_carry[1].flags & kFlagInternal) return -1;
  return (c->h_carry[1].flags & kFlagUtf8) ? 0 : 1;
}

extern "C" int sjb200_validate_utf8_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, void *stream) {
  if (sjb200_validate_utf8_dev_enqueue(c, d_buf, len, stream) != SJB200_SUCCESS) return -1;
  return sjb200_validate_utf8_dev_finish(c);
}

// =============================================================================== host pointers
namespace {

// host staging: input buffer on the device sized to the capacity (+ slack so the last 16-byte vector load is in bounds)
bool ensure_input(sjb200_ctx *c, size_t len) {
  const size_t need = std::max(len, c->capacity) + 256;
  if (c->d_in_bytes >= need) return true;
  cudaFree(c->d_in); c->d_in = nullptr; c->d_in_bytes = 0;
  if (!dev_alloc(c, &c->d_in, need, "cudaMalloc(input)")) return false;
  c->d_in_bytes = need;
  return true;
}
bool ensure_index(sjb200_ctx *c, size_t len) {
  const size_t need = index_words(std::max(len, c->capacity));
  if (c->d_idx_words >= need) return true;
  cudaFree(c->d_idx); c->d_idx = nullptr; c->d_idx_words = 0;
  if (!dev_alloc(c, &c->d_idx, need, "cudaMalloc(index)")) return false;
  c->d_idx_words = need;
  return true;
}
bool ensure_output(sjb200_ctx *c, size_t len) {
  const size_t need = len + 256;
  if (c->d_out_bytes >= need) return true;
  cudaFree(c->d_out); c->d_out = nullptr; c->d_out_bytes = 0;
  if (!dev_alloc(c, &c->d_out, need, "cudaMalloc(output)")) return false;
  c->d_out_bytes = need;
  return true;
}

// page-locked staging ring + copy threads for pageable input (created at the first large host-pointer call)
bool ensure_ring(sjb200_ctx *c, size_t slot_bytes) {
  const int slots = int(c->opt_ring_slots);
  if (c->h_ring && c->ring_slot_bytes >= slot_bytes && c->ring_slots == slots) return true;
  if (c->h_ring) { cudaFreeHost(c->h_ring); c->h_ring = nullptr; c->ring_slot_bytes = 0; c->ring_slots = 0; }
  void *q = nullptr;
  if (!ok(c, cudaMallocHost(&q, slot_bytes * size_t(slots)), "cudaMallocHost(ring)")) return false;
  c->h_ring = static_cast<uint8_t *>(q);
  c->ring_slot_bytes = slot_bytes;
  c->ring_slots = slots;
  while (c->ring_events.size() < size_t(slots)) {
    cudaEvent_t e;
    if (!ok(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "event")) return false;
    c->ring_events.push_back(e);
  }
  return true;
}
bool ensure_pool(sjb200_ctx *c) {
  if (!c->pool) c->pool = new (std::nothrow) CopyPool();
  return c->pool && c->pool->start(int(c->opt_copy_threads));
}

// The host-pointer pipeline.  The document goes to the device chunk by chunk; one scan launch per chunk is chained
// behind its copy (scanner state and output offset travel through d_carry[k] -> d_carry[k+1], flags accumulate);
// later chunks are copied while earlier ones are scanned:  stage(k+2) | H2D(k+1) | scan(k) [| D2H(k-1)].
//   input:  page-locked caller memory -> copied from where it lies; pageable -> through the staging ring (copy threads),
//           small documents straight through the driver.
//   output: stage 1 into a page-locked, mapped caller array (what the plug-in and the Python mirror register) -> the
//           scan kernels store the indexes there themselves (d_idx is then the device alias of host_out and nothing
//           comes back through the copy engine); otherwise each chunk's output is copied back as soon as its launch is done.
// elt = bytes per output element (4 for indexes, 1 for minify, 0 = no output to bring back).
bool scan_host_document(sjb200_ctx *c, int kind, const uint8_t *buf, size_t len, uint32_t *d_idx, uint8_t *d_dst, void *host_out,
                        size_t elt, bool direct_out, int *final_slot) {
  size_t chunk = size_t(c->opt_chunk_bytes);
  const size_t min_chunk = ((len / (kCarrySlots - 8)) / (2 * kTileBytes) + 1) * (2 * kTileBytes);  // at most kCarrySlots-1 chunks
  if (chunk < min_chunk) chunk = min_chunk;
  // chunk boundaries: the first chunks are small and double up to the full size, so that the copy engine and the first
  // scan start early (what precedes the first launch is not overlapped with anything), then equal chunks to the end
  std::vector<size_t> bounds;
  bounds.push_back(0);
  for (size_t c0 = std::min<size_t>(chunk, size_t(c->opt_first_chunk_bytes)); bounds.back() < len;) {
    bounds.push_back(std::min(len, bounds.back() + c0));
    c0 = std::min(chunk, c0 * 2);
  }
  const size_t nchunks = bounds.size() - 1;
  const bool drain = !direct_out && elt != 0 && host_out != nullptr;
  while (c->chunk_events.size() < 2 * nchunks) {
    cudaEvent_t e;
    if (!ok(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "event")) return false;
    c->chunk_events.push_back(e);
  }
  // where does the input come from?
  int in_path = 0;
  {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, buf) == cudaSuccess) {
      if (attr.type == cudaMemoryTypeHost) in_path = 2;
    } else {
      (void)cudaGetLastError();
    }
    if (in_path == 0 && c->opt_copy_threads > 0 && len >= size_t(c->opt_stage_min_bytes) && ensure_ring(c, chunk) && ensure_pool(c)) in_path = 1;
  }
  c->last_input_path = in_path;
  c->last_output_path = direct_out ? 1 : 0;
  CUtensorMap map;
  bool tma = false;
  map_for(c, kind, &map, c->d_in, len, &tma);
  // calls are synchronous, so no earlier kernel still reads d_in when the first copy lands
  auto launch_chunk = [&](size_t k, const uint8_t *src) -> bool {
    const size_t off = bounds[k];
    const size_t bytes = bounds[k + 1] - off;
    cudaEvent_t copied = c->chunk_events[2 * k], scanned = c->chunk_events[2 * k + 1];
    if (!ok(c, cudaMemcpyAsync(c->d_in + off, src, bytes, cudaMemcpyHostToDevice, c->copy_stream), "H2D chunk") ||
        !ok(c, cudaEventRecord(copied, c->copy_stream), "event record") || !ok(c, cudaStreamWaitEvent(c->stream, copied, 0), "wait event"))
      return false;
    const bool last = (k + 1 == nchunks);
    if (c->opt_host_skip_scan) return true;
    if (!enqueue_scan(c, kind, &map, tma, c->d_in, len, uint32_t(off / kTileBytes), tiles_of(bytes), last, 0x20202020u, d_idx, d_dst,
                      k == 0 ? -1 : int(k), c->stream, int(k + 1), false, nullptr, c->h_carry + k + 1))
      return false;
    if (!use_scan4(c, kind) &&  // scan4 mirrors its result to the pinned host slot itself
        !ok(c, cudaMemcpyAsync(c->h_carry + k + 1, c->d_carry + k + 1, sizeof(Carry), cudaMemcpyDeviceToHost, c->stream), "D2H carry"))
      return false;
    return !drain || ok(c, cudaEventRecord(scanned, c->stream), "event record");
  };
  if (in_path == 1) {
    CopyPool &pool = *c->pool;
    const int slots = c->ring_slots;
    pool.begin(buf, bounds.data(), nchunks, c->h_ring, c->ring_slot_bytes, slots);
    pool.allow(size_t(slots));
    size_t issued = 0, released = 0;  // chunks handed to the copy engine / known to have left their slot
    uint32_t idle = 0;
    bool good = true;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms_since = [&](std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double, std::milli>(now() - t0).count(); };
    c->t_wait_ms = c->t_issue_ms = c->t_sync_ms = 0;
    auto t_mark = now();
    while (good && issued < nchunks) {
      while (released < issued && cudaEventQuery(c->chunk_events[2 * released]) == cudaSuccess) {  // (the chunk's "copied" event: one event per copy on the copy stream)
        released++;
        pool.allow(released + size_t(slots));
      }
      if (pool.chunk_ready(issued)) {
        c->t_wait_ms += ms_since(t_mark);
        t_mark = now();
        good = launch_chunk(issued, c->h_ring + (issued % size_t(slots)) * c->ring_slot_bytes);
        c->t_issue_ms += ms_since(t_mark);
        t_mark = now();
        issued++;
        idle = 0;
      } else if (++idle < 512) {
        SJB200_CPU_RELAX();
      } else {
        std::this_thread::sleep_for(std::chrono::microseconds(10));  // (no unbounded spinning: see sjb200_hostpipe.h)
      }
    }
    (void)cudaGetLastError();  // cudaEventQuery's cudaErrorNotReady is not an error
    pool.end(!good);
    if (!good) return false;
  } else {
    for (size_t k = 0; k < nchunks; k++)
      if (!launch_chunk(k, buf + bounds[k])) return false;
  }
  if (drain) {  // bring each chunk's output back as soon as that chunk is done
    uint64_t have = 0;
    for (size_t k = 0; k < nchunks; k++) {
      if (!ok(c, cudaEventSynchronize(c->chunk_events[2 * k + 1]), "event sync")) return false;
      const uint64_t upto = c->h_carry[k + 1].count;
      if (upto > have) {
        const uint8_t *src = (kind == kIndex) ? reinterpret_cast<const uint8_t *>(d_idx) : d_dst;
        if (!ok(c, cudaMemcpyAsync(static_cast<uint8_t *>(host_out) + have * elt, src + have * elt, size_t(upto - have) * elt,
                                   cudaMemcpyDeviceToHost, c->out_stream), "D2H output"))
          return false;
        have = upto;
      }
    }
  }
  const auto t_sync0 = std::chrono::steady_clock::now();
  if (!ok(c, cudaStreamSynchronize(c->stream), "sync") || (drain && !ok(c, cudaStreamSynchronize(c->out_stream), "sync"))) return false;
  c->t_sync_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_sync0).count();
  // every launch reports (and clears) its own flags: the document's flags are their union
  uint32_t flags = 0;
  for (size_t k = 0; k < nchunks; k++) flags |= c->h_carry[k + 1].flags;
  *c->h_flags = flags;
  *final_slot = int(nchunks);
  return true;
}

// device alias of a caller array the kernels may store into directly: page-locked AND mapped host memory
uint32_t *mapped_alias(sjb200_ctx *c, uint32_t *host_ptr) {
  if (!c->opt_zero_copy_out || !host_ptr) return nullptr;
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, host_ptr) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
  if (attr.type != cudaMemoryTypeHost || attr.devicePointer == nullptr) return nullptr;
  return static_cast<uint32_t *>(attr.devicePointer);
}

}  // namespace

extern "C" int sjb200_stage1(sjb200_ctx *c, const uint8_t *buf, size_t len, int mode, uint32_t *idx_out, uint32_t *n_inout) {
  if (!c || !idx_out || !n_inout) return SJB200_UNEXPECTED_ERROR;
  if (mode < SJB200_REGULAR || mode > SJB200_COMMA_DELIMITED_FINAL) return SJB200_UNEXPECTED_ERROR;
  if (len > c->capacity) return SJB200_CAPACITY;                                  // json_structural_indexer.h L195
  if (len == 0) return SJB200_EMPTY;                                              // L197
  if (mode != SJB200_REGULAR) {                                                   // L198-204
    const size_t k = std::min<size_t>(3, len);
    len = trim_partial_utf8_tail(buf + len - k, k, len);
    if (len == 0) return SJB200_UTF8_ERROR;
  }
  DeviceGuard g(c->device);
  uint32_t *alias = use_scan4(c, kIndex) ? mapped_alias(c, idx_out) : nullptr;
  if (!ensure_input(c, len) || (!alias && !ensure_index(c, len)) || !ensure_desc(c, len)) return SJB200_MEMALLOC;
  int slot = 0;
  if (!scan_host_document(c, kIndex, buf, len, alias ? alias : c->d_idx, nullptr, idx_out, sizeof(uint32_t), alias != nullptr, &slot))
    return SJB200_UNEXPECTED_ERROR;
  FinishInput in;
  in.mode = mode; in.len = len;
  in.count = c->h_carry[slot].count;
  in.state = c->h_carry[slot].state;
  in.flags = *c->h_flags;
  in.sentinels_written = false;
  HostStructuralReader reader(buf, idx_out);
  HostIndexWriter writer(idx_out);
  bool dirty = false;
  return finish_stage1(in, reader, writer, n_inout, buf, idx_out, &dirty);
}

extern "C" int sjb200_minify(sjb200_ctx *c, const uint8_t *buf, size_t len, uint8_t *dst, size_t *dst_len) {
  if (!c || !dst_len) return SJB200_UNEXPECTED_ERROR;
  *dst_len = 0;
  if (len == 0) return SJB200_SUCCESS;
  if (len > kMaxBytes) return SJB200_CAPACITY;
  DeviceGuard g(c->device);
  if (!ensure_input(c, len) || !ensure_output(c, len) || !ensure_desc(c, len)) return SJB200_MEMALLOC;
  int slot = 0;
  // the padded tail is never output, so at most len bytes are written to dst (json_minifier.h L79-95)
  if (!scan_host_document(c, kMinify, buf, len, nullptr, c->d_out, dst, 1, false, &slot)) return SJB200_UNEXPECTED_ERROR;
  if (*c->h_flags & kFlagInternal) return SJB200_UNEXPECTED_ERROR;
  if ((c->h_carry[slot].state >> 1) & 1u) return SJB200_UNCLOSED_STRING;
  *dst_len = size_t(c->h_carry[slot].count);
  return SJB200_SUCCESS;
}

extern "C" int sjb200_validate_utf8(sjb200_ctx *c, const uint8_t *buf, size_t len) {
  if (!c) return 0;
  if (len == 0) return 1;
  if (len > kMaxBytes) {
    // the reference's validate_utf8 has no size limit (only stage 1 is bounded by SIMDJSON_MAXSIZE_BYTES): longer inputs
    // go through as consecutive pieces cut at character boundaries -- validity needs no state beyond that
    const size_t piece = size_t(1) << 30;
    size_t off = 0;
    while (off < len) {
      size_t end = (len - off > piece) ? sjb200_shard_cut(buf, len, off + piece) : len;
      if (end <= off) end = std::min(len, off + piece);  // a run of > 3 continuation bytes: invalid anyway, the piece will say so
      if (sjb200_validate_utf8(c, buf + off, end - off) != 1) return 0;
      off = end;
    }
    return 1;
  }
  DeviceGuard g(c->device);
  if (!ensure_input(c, len)) return 0;
  int slot = 0;
  if (!scan_host_document(c, kUtf8, buf, len, nullptr, nullptr, nullptr, 0, false, &slot)) return 0;
  if (*c->h_flags & kFlagInternal) return 0;
  return (*c->h_flags & kFlagUtf8) ? 0 : 1;
}

// =============================================================================== shards (multi-GPU)
extern "C" int sjb200_stage1_shard_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, uint32_t state_in, int last_shard,
                                       uint32_t *d_idx, sjb200_shard_result *out, void *stream) {
  if (!c || !out) return SJB200_UNEXPECTED_ERROR;
  memset(out, 0, sizeof(*out));
  if (len == 0 || len > kMaxBytes) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (!ensure_desc(c, len)) return SJB200_MEMALLOC;
  CUtensorMap map;
  bool tma = false;
  map_for(c, kIndex, &map, d_buf, len, &tma);
  c->h_carry[0].count = 0; c->h_carry[0].state = state_in & 7u; c->h_carry[0].ttable = 0;
  (void)last_shard;  // every shard checks its own end: cuts are at character boundaries (sjb200_shard_cut)
  c->h_carry[0].flags = 0; c->h_carry[0].reserved = 0;
  if (!ok(c, cudaMemcpyAsync(c->d_carry, c->h_carry, sizeof(Carry), cudaMemcpyHostToDevice, s), "H2D carry") ||
      !enqueue_scan(c, kIndex, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, d_idx, nullptr, 0, s) ||
      !fetch_result(c, s) || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  out->ttable = c->h_carry[1].ttable;
  out->state_out = c->h_carry[1].state;
  out->flags = c->h_carry[1].flags;
  out->count = c->h_carry[1].count;
  return (out->flags & kFlagInternal) ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
}

// Speculative pass of a shard (incoming state 0) without any host synchronisation: the 24-byte result
// {count, state_out, ttable, flags} is written to caller-provided DEVICE memory, ready to be the send buffer of an
// all-gather enqueued behind it on the same stream.
extern "C" int sjb200_stage1_shard_dev_enqueue(sjb200_ctx *c, const uint8_t *d_buf, size_t len, uint32_t *d_idx, void *d_result,
                                               void *stream) {
  if (!c || !d_result || len == 0 || len > kMaxBytes) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (!ensure_desc(c, len)) return SJB200_MEMALLOC;
  CUtensorMap map;
  bool tma = false;
  map_for(c, kIndex, &map, d_buf, len, &tma);
  if (!enqueue_scan(c, kIndex, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, d_idx, nullptr, -1, s, 1, false,
                    static_cast<Carry *>(d_result)))
    return SJB200_UNEXPECTED_ERROR;
  return SJB200_SUCCESS;
}

// =============================================================================== sharded scan with the exchange fused in
// One object per rank.  The exchange window lives in device memory; peers map it through CUDA IPC (one process per GPU,
// the torch.distributed / MPI layout) or directly (several contexts in one process).  A pass = every rank scans its
// shard with the speculated state 0; the scan kernel's last CTA stores the 16-byte record {count, state, transducer,
// flags} into every rank's window over NVLink -- no collective launch.  finish() reads the local window, folds the
// true incoming state and index base, and -- only when somebody's speculation was wrong -- re-scans and runs a second
// round.  Up to kXchgSteps / 2 passes may be in flight per rank (enqueue ... enqueue, finish ... finish).
struct sjb200_comm {
  sjb200_ctx *ctx = nullptr;
  int rank = 0, nranks = 1;
  unsigned long long *window = nullptr;            // [kXchgSteps][2 rounds][kMaxRanks][2]
  unsigned long long *peer[kMaxRanks] = {};        // peer[r] = rank r's window as seen from this device
  bool opened[kMaxRanks] = {};                     // mapped through cudaIpcOpenMemHandle (to be closed)
  bool connected = false;
  unsigned long long *h_rec = nullptr;             // pinned [kMaxRanks][2]
  Carry *d_result = nullptr;                       // [kXchgSteps] the launches' own result blocks
  cudaStream_t poll_stream = nullptr;
  cudaEvent_t done[kXchgSteps] = {};
  struct Step { const uint8_t *d_buf; size_t len; uint32_t *d_idx; cudaStream_t stream; uint32_t seq; int last; } steps[kXchgSteps];
  uint32_t head = 0, tail = 0;                     // passes enqueued / finished
  long poll_timeout_ms = 20000;
};

namespace {
constexpr size_t kWindowWords = size_t(kXchgSteps) * 2 * kMaxRanks * 2;
uint32_t window_slot(uint32_t seq, int round) { return (seq % uint32_t(kXchgSteps)) * 2u + uint32_t(round); }

// wait (host polling, bounded) until every rank's record of (seq, round) is in the local window; records -> comm->h_rec
int comm_collect(sjb200_comm *m, uint32_t seq, int round) {
  sjb200_ctx *c = m->ctx;
  const unsigned long long *src = m->window + size_t(window_slot(seq, round)) * kMaxRanks * 2;
  const auto t0 = std::chrono::steady_clock::now();
  for (;;) {
    if (!ok(c, cudaMemcpyAsync(m->h_rec, src, size_t(m->nranks) * 16, cudaMemcpyDeviceToHost, m->poll_stream), "D2H window") ||
        !ok(c, cudaStreamSynchronize(m->poll_stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->xchg_polls++;
    bool all = true;
    for (int r = 0; r < m->nranks; r++) all = all && xchg_complete(m->h_rec[2 * r], m->h_rec[2 * r + 1], seq);
    if (all) {
      c->xchg_wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      return SJB200_SUCCESS;
    }
    if (std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - t0).count() > m->poll_timeout_ms) {
      c->last_error = "sharded scan: a peer's record did not arrive";
      return SJB200_UNEXPECTED_ERROR;
    }
  }
}
}  // namespace

extern "C" int sjb200_comm_create(sjb200_ctx *c, int rank, int nranks, sjb200_comm **out) {
  if (!c || !out || nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks) return SJB200_UNEXPECTED_ERROR;
  *out = nullptr;
  DeviceGuard g(c->device);
  sjb200_comm *m = new (std::nothrow) sjb200_comm();
  if (!m) return SJB200_MEMALLOC;
  m->ctx = c; m->rank = rank; m->nranks = nranks;
  void *hp = nullptr;
  bool good = dev_alloc(c, &m->window, kWindowWords, "cudaMalloc(window)") &&
              ok(c, cudaMemset(m->window, 0, kWindowWords * sizeof(unsigned long long)), "memset window") &&
              dev_alloc(c, &m->d_result, kXchgSteps, "cudaMalloc(results)") &&
              ok(c, cudaMallocHost(&hp, kMaxRanks * 16), "cudaMallocHost") &&
              ok(c, cudaStreamCreateWithFlags(&m->poll_stream, cudaStreamNonBlocking), "stream");
  m->h_rec = static_cast<unsigned long long *>(hp);
  for (int i = 0; good && i < kXchgSteps; i++) good = ok(c, cudaEventCreateWithFlags(&m->done[i], cudaEventDisableTiming), "event");
  if (!good) { sjb200_comm_destroy(m); return SJB200_MEMALLOC; }
  m->peer[rank] = m->window;
  m->connected = (nranks == 1);
  *out = m;
  return SJB200_SUCCESS;
}

extern "C" void sjb200_comm_destroy(sjb200_comm *m) {
  if (!m) return;
  DeviceGuard g(m->ctx->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < kMaxRanks; r++)
    if (m->opened[r] && m->peer[r]) cudaIpcCloseMemHandle(m->peer[r]);
  cudaFree(m->window); cudaFree(m->d_result);
  if (m->h_rec) cudaFreeHost(m->h_rec);
  if (m->poll_stream) cudaStreamDestroy(m->poll_stream);
  for (auto e : m->done) if (e) cudaEventDestroy(e);
  (void)cudaGetLastError();
  delete m;
}

extern "C" int sjb200_comm_get_handle(sjb200_comm *m, void *handle) {
  if (!m || !handle) return SJB200_UNEXPECTED_ERROR;
  static_assert(sizeof(cudaIpcMemHandle_t) == SJB200_COMM_HANDLE_BYTES, "handle size");
  DeviceGuard g(m->ctx->device);
  cudaIpcMemHandle_t h;
  if (!ok(m->ctx, cudaIpcGetMemHandle(&h, m->window), "cudaIpcGetMemHandle")) return SJB200_UNEXPECTED_ERROR;
  memcpy(handle, &h, sizeof(h));
  return SJB200_SUCCESS;
}

extern "C" int sjb200_comm_connect(sjb200_comm *m, const void *handles) {
  if (!m || !handles) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(m->ctx->device);
  for (int r = 0; r < m->nranks; r++) {
    if (r == m->rank || m->peer[r]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const uint8_t *>(handles) + size_t(r) * sizeof(h), sizeof(h));
    void *q = nullptr;
    if (!ok(m->ctx, cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle")) return SJB200_UNEXPECTED_ERROR;
    m->peer[r] = static_cast<unsigned long long *>(q);
    m->opened[r] = true;
  }
  m->connected = true;
  return SJB200_SUCCESS;
}

// ranks that live in ONE process (several contexts, same or different devices): plain pointers, peer access enabled
extern "C" int sjb200_comm_connect_local(sjb200_comm *m, sjb200_comm *const *all) {
  if (!m || !all) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(m->ctx->device);
  for (int r = 0; r < m->nranks; r++) {
    if (!all[r] || all[r]->nranks != m->nranks || all[r]->rank != r) return SJB200_UNEXPECTED_ERROR;
    if (all[r]->ctx->device != m->ctx->device) {
      cudaError_t e = cudaDeviceEnablePeerAccess(all[r]->ctx->device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { ok(m->ctx, e, "cudaDeviceEnablePeerAccess"); return SJB200_UNEXPECTED_ERROR; }
      (void)cudaGetLastError();
    }
    m->peer[r] = all[r]->window;
  }
  m->connected = true;
  return SJB200_SUCCESS;
}

extern "C" int sjb200_stage1_sharded_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx, void *stream) {
  if (!m || !m->connected || !d_shard || !d_idx || len == 0 || len > kMaxBytes) return SJB200_UNEXPECTED_ERROR;
  if (m->head - m->tail >= uint32_t(kXchgSteps / 2)) return SJB200_CAPACITY;  // too many passes in flight: finish some first
  sjb200_ctx *c = m->ctx;
  if (!use_scan4(c, kIndex)) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  const auto t_enq = std::chrono::steady_clock::now();
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (!ensure_desc(c, len)) return SJB200_MEMALLOC;
  const uint32_t seq = m->head + 1;  // tags start at 1: a zeroed window never matches
  XchgTarget x;
  for (int r = 0; r < kMaxRanks; r++) x.peer[r] = m->peer[r];
  x.nranks = uint32_t(m->nranks); x.rank = uint32_t(m->rank); x.slot = window_slot(seq, 0); x.seq = seq;
  CUtensorMap map;
  bool tma = false;
  map_for(c, kIndex, &map, d_shard, len, &tma);
  sjb200_comm::Step &st = m->steps[m->head % uint32_t(kXchgSteps)];
  st.d_buf = d_shard; st.len = len; st.d_idx = d_idx; st.stream = s; st.seq = seq; st.last = last_shard;
  if (!enqueue_scan(c, kIndex, &map, tma, d_shard, len, 0, tiles_of(len), true, 0x20202020u, d_idx, nullptr, -1, s, 1, false,
                    m->d_result + (m->head % uint32_t(kXchgSteps)), nullptr, &x) ||
      !ok(c, cudaEventRecord(m->done[m->head % uint32_t(kXchgSteps)], s), "event record"))
    return SJB200_UNEXPECTED_ERROR;
  m->head++;
  c->xchg_enqueue_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enq).count();
  return SJB200_SUCCESS;
}

extern "C" int sjb200_stage1_sharded_finish(sjb200_comm *m, sjb200_sharded_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  memset(out, 0, sizeof(*out));
  const sjb200_comm::Step st = m->steps[m->tail % uint32_t(kXchgSteps)];
  const uint32_t slot_i = m->tail % uint32_t(kXchgSteps);
  m->tail++;
  const auto t_ev = std::chrono::steady_clock::now();
  if (!ok(c, cudaEventSynchronize(m->done[slot_i]), "event sync")) return SJB200_UNEXPECTED_ERROR;  // own scan (and its stores) done
  c->xchg_evsync_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_ev).count();
  int rc = comm_collect(m, st.seq, 0);
  if (rc != SJB200_SUCCESS) return rc;
  uint32_t tt[kMaxRanks], flags_all = 0;
  bool any_wrong = false;
  uint32_t state = 0, my_state = 0;
  for (int r = 0; r < m->nranks; r++) {
    tt[r] = uint32_t(m->h_rec[2 * r + 1] >> 8) & 0x3Fu;
    if (r == m->rank) my_state = state;
    if (state != 0) any_wrong = true;
    state = tt_apply(tt[r], state);
  }
  out->state_in = my_state;
  out->state_out = tt_apply(tt[m->rank], my_state);
  out->final_state = state;
  uint64_t my_count = xchg_count(m->h_rec[2 * m->rank]);
  uint32_t my_flags = uint32_t(m->h_rec[2 * m->rank + 1] >> 16) & 0xFFu;
  if (any_wrong) {
    c->xchg_second_rounds++;
    // second round: ranks whose speculation failed scan again with their true state; everybody republishes
    if (my_state != 0) {
      sjb200_shard_result sr;
      rc = sjb200_stage1_shard_dev(c, st.d_buf, st.len, my_state, st.last, st.d_idx, &sr, st.stream);
      if (rc != SJB200_SUCCESS) return rc;
      my_count = sr.count;
      my_flags = sr.flags;
      out->rescanned = 1;
    }
    ScanParams p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < kMaxRanks; r++) p.xchg_peer[r] = m->peer[r];
    p.xchg_nranks = uint32_t(m->nranks); p.xchg_rank = uint32_t(m->rank); p.xchg_slot = window_slot(st.seq, 1); p.xchg_seq = st.seq;
    if (!ok(c, launch_xchg_post(p, xchg_word0(st.seq, my_count), xchg_word1(st.seq, out->state_out, tt[m->rank], my_flags), st.stream), "xchg post") ||
        !ok(c, cudaStreamSynchronize(st.stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->launches++;
    rc = comm_collect(m, st.seq, 1);
    if (rc != SJB200_SUCCESS) return rc;
  }
  uint64_t base = 0, total = 0;
  for (int r = 0; r < m->nranks; r++) {
    const uint64_t cnt = xchg_count(m->h_rec[2 * r]);
    if (r < m->rank) base += cnt;
    total += cnt;
    flags_all |= uint32_t(m->h_rec[2 * r + 1] >> 16) & 0xFFu;
  }
  out->count = my_count;
  out->base = base;
  out->total_count = total;
  out->flags = my_flags;
  out->flags_all = flags_all;
  return ((my_flags | flags_all) & kFlagInternal) ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
}

extern "C" int sjb200_stage1_sharded(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx,
                                     sjb200_sharded_result *out, void *stream) {
  int rc = sjb200_stage1_sharded_enqueue(m, d_shard, len, last_shard, d_idx, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_stage1_sharded_finish(m, out);
}

extern "C" uint32_t sjb200_fold_state(const uint32_t *ttables, int nshards_before) {
  uint32_t state = 0;
  for (int i = 0; i < nshards_before; i++) state = tt_apply(ttables[i], state);
  return state;
}

extern "C" size_t sjb200_shard_cut(const uint8_t *buf, size_t len, size_t nominal) {
  if (nominal >= len) return len;
  size_t cut = nominal;
  for (int k = 0; k < 3 && cut > 0 && (buf[cut] & 0xC0) == 0x80; k++) cut--;
  return cut;
}

extern "C" size_t sjb200_shard_cut_line(const uint8_t *buf, size_t len, size_t nominal, size_t window) {
  if (nominal >= len) return len;
  const size_t lo = nominal > window ? nominal - window : 0;
  for (size_t cut = nominal; cut > lo; cut--)
    if (buf[cut - 1] == 0x0A) return cut;
  return sjb200_shard_cut(buf, len, nominal);
}
