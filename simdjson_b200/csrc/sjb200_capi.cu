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
  // [0] the launch's flags, [1 + slot] the flags of the document whose result goes to carry slot `slot`, [1 + kCarrySlots]
  // the flags of a launch of parity 1 (launch_flags)
  uint32_t *d_flags = nullptr;
  uint32_t *d_ticket = nullptr;  // [parity][4]
  unsigned long long *d_count_desc = nullptr;  // [parity][desc_tiles]
  size_t desc_tiles = 0;
  unsigned long long *d_stamps = nullptr; size_t stamps_cap = 0; size_t stamps_used = 0;  // option launch_stamps: [launch][2]
  StreamFinish *d_sfin = nullptr;  // [kCarrySlots] results of the device-side streaming epilogue
  uint32_t *d_doc_scratch = nullptr; size_t doc_scratch_words = 0; uint32_t *d_ndocs = nullptr;
  void *d_tok_scratch = nullptr; size_t tok_scratch_bytes = 0; TokenTotals *d_tok_tot = nullptr;  // stage-2-lite (sjb200_tape.cu)
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
  std::vector<uint32_t> ev_docs;                 // [i] documents launch i scanned
  size_t ev_used = 0;
  uint32_t ev_last_docs = 1;                     // ... the launch around ev_k0 / ev_k1
  // multi-document stage-1 launches: per group a DocEntry table and the documents' tensor maps, encoded for a whole
  // batch round into pinned memory, copied group by group ahead of the launches
  uint8_t *h_doctab = nullptr; uint8_t *d_doctab = nullptr; size_t doctab_bytes = 0;
  long opt_debug_timeline = 0;
  long opt_pdl = 1, opt_launch_stamps = 0;
  unsigned long long *d_debug = nullptr; size_t debug_tiles = 0; uint32_t debug_last_tiles = 0;
  unsigned long long launches = 0;               // kernels of ours launched by this context
  PFN_encodeTiled encode = nullptr;
  TmapCacheEntry tmap_cache[kTmapCacheEntries];  // make_tensor_map
  // host-pointer pipeline: ring of page-locked staging slots filled by copy threads (sjb200_hostpipe.h)
  uint8_t *h_ring = nullptr; size_t ring_slot_bytes = 0; int ring_slots = 0;
  std::vector<cudaEvent_t> ring_events;
  CopyPool *pool = nullptr;
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

// look-back descriptors: sized for the capacity, zeroed once (epoch tags make them reusable).  `need` descriptors: one per
// tile is more than one per element.  Two sets, one per launch parity (launch_desc).
bool ensure_desc_n(sjb200_ctx *c, size_t need) {
  need = std::max<size_t>(need, 1);
  if (need <= c->desc_tiles) return true;
  cudaFree(c->d_count_desc); c->d_count_desc = nullptr;
  c->desc_tiles = 0;
  const size_t n = std::max(need, size_t(tiles_of(c->capacity)) + 1);
  if (!dev_alloc(c, &c->d_count_desc, 2 * n, "cudaMalloc(count_desc)")) return false;
  if (!ok(c, cudaMemsetAsync(c->d_count_desc, 0, 2 * n * sizeof(unsigned long long), c->stream), "memset desc")) return false;
  if (!ok(c, cudaStreamSynchronize(c->stream), "sync")) return false;
  c->desc_tiles = n;
  c->epoch = 0;
  return true;
}
bool ensure_desc(sjb200_ctx *c, size_t len) { return ensure_desc_n(c, tiles_of(len)); }

// The wipe at the wrap of the 18-bit tag is ordered on the LAUNCH stream (a context is used on one stream at a time,
// see sjb200.h): kernels queued earlier on it finish before the wipe, the next launch starts after it.  *wiped: the
// wipe was queued (it then sits between the previous launch and the next one).
bool next_epoch(sjb200_ctx *c, cudaStream_t launch_stream, uint32_t *epoch, bool *wiped = nullptr) {
  c->epoch++;
  if (wiped) *wiped = false;
  if (c->epoch >= (1u << 18)) {
    if (!ok(c, cudaMemsetAsync(c->d_count_desc, 0, 2 * c->desc_tiles * sizeof(unsigned long long), launch_stream), "memset desc")) return false;
    c->epoch = 1;
    if (wiped) *wiped = true;
  }
  *epoch = c->epoch;
  return true;
}

// The scratch a stage-1 launch re-arms for the next one -- ticket block, launch flags word, look-back descriptors -- in
// two sets.  Two consecutive scan launches of a batch call may run at once (programmatic dependent launch): they use
// alternate sets, and a launch starts only after the one two before it has completed.  Every other launch uses set 0.
uint32_t *launch_ticket(sjb200_ctx *c, int parity) { return c->d_ticket + 4 * parity; }
uint32_t *launch_flags(sjb200_ctx *c, int parity) { return parity ? c->d_flags + 1 + kCarrySlots : c->d_flags; }
unsigned long long *launch_desc(sjb200_ctx *c, int parity) { return c->d_count_desc + size_t(parity) * c->desc_tiles; }

// the tensor map every scan kernel reads through: 4 KiB boxes of 32 rows of 128 bytes
bool make_tensor_map(sjb200_ctx *c, CUtensorMap *map, const uint8_t *d_buf, size_t len, bool *usable) {
  memset(map, 0, sizeof(*map));
  *usable = false;
  const uint64_t rows = len / 128;
  if (!c->opt_use_tma || c->encode == nullptr || rows == 0) return true;
  if ((reinterpret_cast<uintptr_t>(d_buf) & 15u) != 0) return true;  // TMA needs a 16-byte aligned base
  // A map is a function of (base, rows) alone; re-encoding it costs ~1 us of host time per document, which a batch
  // call of many documents pays before its first launch.  Recently encoded maps are kept in a small direct-mapped cache.
  const uintptr_t key = reinterpret_cast<uintptr_t>(d_buf);
  TmapCacheEntry &ce = c->tmap_cache[((key >> 4) ^ (key >> 12) ^ rows) % kTmapCacheEntries];
  if (ce.base == d_buf && ce.rows == rows) {
    *map = ce.map;
    *usable = true;
    return true;
  }
  cuuint64_t dims[2] = {128, rows};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {128, (cuuint32_t)kScan4BoxRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = c->encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t *>(d_buf), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    c->last_error = "cuTensorMapEncodeTiled failed (" + std::to_string(int(r)) + "); using plain loads";
    return true;
  }
  ce.base = d_buf;
  ce.rows = rows;
  ce.map = *map;
  *usable = true;
  return true;
}

int grid_cap(sjb200_ctx *c) {
  if (c->grid4 == 0) c->grid4 = scan4_max_ctas_per_sm() * c->sm_count;
  return c->opt_grid > 0 ? int(c->opt_grid) : c->grid4;
}
int grid_for(sjb200_ctx *c, uint32_t nelements) {
  if (c->opt_force_grid > 0) return int(c->opt_force_grid);  // tuning: a full grid even for a tiny document (measures the fixed cost of a launch)
  return int(std::max<uint32_t>(1, std::min<uint32_t>(uint32_t(grid_cap(c)), nelements)));
}

// where a sharded launch publishes its record (sjb200_comm), and the kind the record carries
struct XchgTarget {
  unsigned long long *peer[kMaxRanks];
  uint32_t nranks, rank, slot, seq, kind;
};

// Option time_kernel: events around one scan launch.  time_begin records the first one and returns the second (null:
// not timed); time_end records the second.  `docs` = documents the launch scanned: kernel_ms / kernel_ms_mean report
// its duration per document.
cudaEvent_t time_begin(sjb200_ctx *c, cudaStream_t stream) {
  if (!c->opt_time_kernel) return nullptr;
  if (c->ev_used + 2 > c->ev_pool.size() && c->ev_pool.size() < 4096) {
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    c->ev_pool.push_back(a); c->ev_pool.push_back(b);
    c->ev_docs.push_back(1);
  }
  if (c->ev_used + 2 > c->ev_pool.size()) return nullptr;
  cudaEventRecord(c->ev_pool[c->ev_used], stream);
  c->ev_used += 2;
  return c->ev_pool[c->ev_used - 1];
}
void time_end(sjb200_ctx *c, cudaStream_t stream, cudaEvent_t e1, bool launched, uint32_t docs) {
  if (!e1) return;
  cudaEventRecord(e1, stream);
  c->ev_docs[c->ev_used / 2 - 1] = docs;
  c->ev_k0 = c->ev_pool[c->ev_used - 2]; c->ev_k1 = e1; c->ev_valid = launched; c->ev_last_docs = docs;
}

// Enqueue the scan of document tiles [tile_begin, tile_begin+ntiles) of (d_buf,len).
bool enqueue_scan(sjb200_ctx *c, int kind, const CUtensorMap *map, bool tma, const uint8_t *d_buf, size_t len, uint32_t tile_begin,
                  uint32_t ntiles, bool has_last_tile, uint32_t prev_word, uint32_t *d_idx, uint8_t *d_dst, int carry_in_slot,
                  cudaStream_t stream, int carry_out_slot = -1, bool write_sentinels = false, Carry *external_out = nullptr,
                  Carry *host_out = nullptr, const XchgTarget *xchg = nullptr, bool timed = true) {
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
  p.carry_out_host = host_out;
  p.flags = c->d_flags;
  p.count_desc = c->d_count_desc;
  p.ticket = c->d_ticket;
  if (xchg) {  // both kernels publish the record (scan4: stage 1 and minify; utf8v2: validate_utf8)
    for (int r = 0; r < kMaxRanks; r++) p.xchg_peer[r] = xchg->peer[r];
    p.xchg_nranks = xchg->nranks; p.xchg_rank = xchg->rank; p.xchg_slot = xchg->slot; p.xchg_seq = xchg->seq; p.xchg_kind = xchg->kind;
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
  cudaEvent_t e1 = timed ? time_begin(c, stream) : nullptr;
  bool launched;
  if (kind == kUtf8) {  // validate_utf8: utf8v2 (sjb200_utf8.cuh); stage 1 and minify: scan4 (sjb200_scan4.cuh)
    if (c->grid_u == 0) c->grid_u = utf8v2_max_ctas_per_sm() * c->sm_count;
    const uint64_t nblocks = (uint64_t(ntiles) * kTileBytes + 4095) / 4096;
    const uint64_t want = (nblocks + uint64_t(utf8v2_warps_per_cta()) - 1) / uint64_t(utf8v2_warps_per_cta());
    const int grid = c->opt_force_grid > 0 ? int(c->opt_force_grid) : int(std::max<uint64_t>(1, std::min<uint64_t>(uint64_t(c->opt_grid > 0 ? c->opt_grid : c->grid_u), want)));
    launched = ok(c, launch_utf8v2(map, p, grid, stream), "launch utf8v2");
  } else {
    const uint32_t tpe = uint32_t(scan4_tiles_per_element());
    const uint32_t nelem = (ntiles + tpe - 1) / tpe;
    launched = ok(c, launch_scan4(map, p, grid_for(c, nelem), kind == kMinify ? 2 : 0, stream), "launch scan4");
  }
  time_end(c, stream, e1, launched, 1);
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
              dev_alloc(c, &c->d_carry, kCarrySlots, "cudaMalloc(carry)") && dev_alloc(c, &c->d_flags, 2 + kCarrySlots, "cudaMalloc(flags)") &&
              dev_alloc(c, &c->d_ticket, 8, "cudaMalloc(ticket)") &&
              ok(c, cudaMemset(c->d_ticket, 0, 8 * sizeof(uint32_t)), "memset ticket") &&
              ok(c, cudaMemset(c->d_flags, 0, (2 + kCarrySlots) * sizeof(uint32_t)), "memset flags");
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
  cudaFree(c->d_carry); cudaFree(c->d_flags); cudaFree(c->d_ticket); cudaFree(c->d_sfin); cudaFree(c->d_doc_scratch); cudaFree(c->d_ndocs); cudaFree(c->d_tok_scratch); cudaFree(c->d_tok_tot); cudaFree(c->d_tails); cudaFree(c->d_tail_ptrs); cudaFree(c->d_debug); cudaFree(c->d_doctab); cudaFree(c->d_stamps);
  if (c->h_doctab) cudaFreeHost(c->h_doctab);
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

extern "C" long sjb200_get_launch_stamps(sjb200_ctx *c, unsigned long long *out, size_t max_launches) {
  if (!c || !c->d_stamps || !out) return 0;
  DeviceGuard g(c->device);
  const size_t n = std::min(max_launches, c->stamps_used);
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(out, c->d_stamps, n * 16, cudaMemcpyDeviceToHost) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
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
  if (!strcmp(key, "kernel_ms")) {  // duration of the last scan kernel per document it scanned (needs option time_kernel=1 and a finished call)
    if (!c->ev_valid) return -1.0;
    DeviceGuard g(c->device);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev_k0, c->ev_k1) != cudaSuccess) { (void)cudaGetLastError(); return -1.0; }
    return double(ms) / double(c->ev_last_docs);
  }
  if (!strcmp(key, "kernel_ms_mean")) {  // scan kernel time per document, over the kernels launched since the previous query
    DeviceGuard g(c->device);
    double sum = 0;
    size_t n = 0;
    for (size_t i = 0; i + 1 < c->ev_used; i += 2) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, c->ev_pool[i], c->ev_pool[i + 1]) == cudaSuccess) { sum += ms; n += c->ev_docs[i / 2]; } else (void)cudaGetLastError();
    }
    c->ev_used = 0;
    c->ev_valid = false;
    return n ? sum / double(n) : -1.0;
  }
  if (!strcmp(key, "launches")) return double(c->launches);
  if (!strcmp(key, "grid_index")) return double(grid_for(c, 0xFFFFFFFFu));
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
  else if (!strcmp(key, "pdl")) c->opt_pdl = value ? 1 : 0;
  else if (!strcmp(key, "launch_stamps")) c->opt_launch_stamps = value ? 1 : 0;
  else if (!strcmp(key, "chunk_bytes")) c->opt_chunk_bytes = std::max<long>(2 * kTileBytes, (value / (2 * kTileBytes)) * (2 * kTileBytes));
  else if (!strcmp(key, "force_grid")) c->opt_force_grid = value;
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
// The checks before a device-resident stage-1 scan and the trim of a partial UTF-8 tail (json_structural_indexer.h
// L195-204).  False: the call ends here, with pc.early_error.
bool stage1_prepare(sjb200_ctx *c, PendingCall &pc, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, cudaStream_t s, int slot,
                    const uint8_t *tail3 /* host copy of the last min(3, len) bytes, when the caller fetched it */) {
  pc = PendingCall();
  pc.kind = kIndex; pc.mode = mode; pc.d_buf = d_buf; pc.d_idx = d_idx; pc.stream = s; pc.len = len; pc.carry_slot = slot;
  if (mode < SJB200_REGULAR || mode > SJB200_COMMA_DELIMITED_FINAL) { pc.early_error = SJB200_UNEXPECTED_ERROR; return false; }
  if (len > c->capacity) { pc.early_error = SJB200_CAPACITY; return false; }   // json_structural_indexer.h L195
  if (len == 0) { pc.early_error = SJB200_EMPTY; return false; }                // L197
  if (mode != SJB200_REGULAR) {                                                 // L198-204
    const size_t k = std::min<size_t>(3, len);
    if (!tail3) {
      if (!ok(c, cudaMemcpyAsync(c->h_small, d_buf + len - k, k, cudaMemcpyDeviceToHost, s), "D2H tail") ||
          !ok(c, cudaStreamSynchronize(s), "sync"))
        { pc.early_error = SJB200_UNEXPECTED_ERROR; return false; }
      tail3 = c->h_small;
    }
    len = trim_partial_utf8_tail(tail3, k, len);
    pc.len = len;
    if (len == 0) { pc.early_error = SJB200_UTF8_ERROR; return false; }
  }
  return true;
}

// whitespace-separated streams: the rest of finish() (find_next_document_index, the final fix-up) runs on the device
// right behind the scan -- no host round trip between the two (sjb200_docs.cu).  Returns whether it queued anything.
bool stage1_stream_epilogue(sjb200_ctx *c, PendingCall &pc) {
  if (pc.mode == SJB200_STREAMING_PARTIAL || pc.mode == SJB200_STREAMING_FINAL) {
    c->launches++;
    const int slot = pc.carry_slot;
    if (!ok(c, launch_stream_finish(pc.d_buf, pc.d_idx, c->d_carry + slot, uint32_t(pc.len), pc.mode, c->d_sfin + slot, c->h_sfin + slot, pc.stream), "stream finish"))
      pc.early_error = SJB200_UNEXPECTED_ERROR;
    return true;
  }
  return false;
}

// enqueue one device-resident stage-1 scan; its {count,state,flags} come back in h_carry[slot]
void stage1_enqueue_into(sjb200_ctx *c, PendingCall &pc, const uint8_t *d_buf, size_t len, int mode, uint32_t *d_idx, cudaStream_t s, int slot) {
  if (!stage1_prepare(c, pc, d_buf, len, mode, d_idx, s, slot, nullptr)) return;
  len = pc.len;
  if (!ensure_desc(c, len)) { pc.early_error = SJB200_MEMALLOC; return; }
  CUtensorMap map;
  bool tma = false;
  make_tensor_map(c, &map, d_buf, len, &tma);
  // the kernel stores its result in the pinned host mirror itself
  if (!enqueue_scan(c, kIndex, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, d_idx, nullptr, -1, s, slot, true, nullptr,
                    c->h_carry + slot))
    { pc.early_error = SJB200_UNEXPECTED_ERROR; return; }
  stage1_stream_epilogue(c, pc);
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

namespace {
bool ranges_overlap(const void *a, size_t an, const void *b, size_t bn) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + bn && y < x + an;
}
size_t out_bytes(const PendingCall &pc) { return 4 * (pc.len + 3); }  // at most len structurals + 3 sentinels

// Enqueue the scans of the prepared calls (those without an early error), consecutive documents grouped into one
// multi-document launch each.  A group ends before a document that reads or writes memory an earlier document of the
// group writes, or writes memory it reads: the launches then keep the order of a one-by-one loop.  The tables of all
// groups are encoded into pinned memory and go to the device in one copy before the first launch, so that nothing sits
// on the stream between two scan launches: a multi-document launch right behind another one starts while that one
// still runs (programmatic dependent launch, option pdl) and waits for it only before an access that could conflict
// (sjb200_scan4.cuh, wait_previous_launch).  Nothing waits for the device.  With time_kernel, one event pair spans all
// launches of the call (overlapping launches have no duration of their own).
int enqueue_doc_groups(sjb200_ctx *c, std::vector<PendingCall> &calls, cudaStream_t s) {
  constexpr uint64_t kMaxGroupElems = 1u << 20;  // 64 GiB of input; 8 MiB of look-back descriptors
  const uint32_t tpe = uint32_t(scan4_tiles_per_element());
  auto elems_of = [&](const PendingCall &pc) { return uint64_t((tiles_of(pc.len) + tpe - 1) / tpe); };
  std::vector<std::vector<int>> groups;
  uint64_t g_elems = 0, max_elems = 0;
  for (int i = 0; i < int(calls.size()); i++) {
    const PendingCall &pc = calls[size_t(i)];
    if (pc.early_error >= 0) continue;
    bool split = groups.empty() || groups.back().size() == size_t(kMaxLaunchDocs) || g_elems + elems_of(pc) > kMaxGroupElems;
    for (size_t k = 0; !split && k < groups.back().size(); k++) {
      const PendingCall &q = calls[size_t(groups.back()[k])];
      split = ranges_overlap(pc.d_buf, pc.len, q.d_idx, out_bytes(q)) || ranges_overlap(pc.d_idx, out_bytes(pc), q.d_idx, out_bytes(q)) ||
              ranges_overlap(pc.d_idx, out_bytes(pc), q.d_buf, q.len);
    }
    if (split) { groups.emplace_back(); g_elems = 0; }
    groups.back().push_back(i);
    g_elems += elems_of(pc);
    max_elems = std::max(max_elems, g_elems);
  }
  if (groups.empty()) return SJB200_SUCCESS;
  if (!ensure_desc_n(c, max_elems)) return SJB200_MEMALLOC;
  // table layout of group g at offset off[g]: ndocs DocEntry, then ndocs tensor maps (64-byte aligned)
  std::vector<size_t> off(groups.size() + 1, 0);
  for (size_t g = 0; g < groups.size(); g++) {
    const size_t n = groups[g].size() > 1 ? groups[g].size() : 0;  // a group of one is an ordinary single-document launch
    off[g + 1] = off[g] + ((n * sizeof(DocEntry) + 127) & ~size_t(127)) + n * sizeof(CUtensorMap);
  }
  if (off.back() > c->doctab_bytes) {
    if (c->h_doctab) cudaFreeHost(c->h_doctab);
    cudaFree(c->d_doctab);
    c->h_doctab = nullptr; c->d_doctab = nullptr; c->doctab_bytes = 0;
    void *hp = nullptr;
    if (!ok(c, cudaMallocHost(&hp, off.back()), "cudaMallocHost(doc tables)") || !dev_alloc(c, &c->d_doctab, off.back(), "cudaMalloc(doc tables)"))
      return SJB200_MEMALLOC;
    c->h_doctab = static_cast<uint8_t *>(hp);
    c->doctab_bytes = off.back();
  }
  static_assert(sizeof(DocEntry) == 64 && sizeof(CUtensorMap) == 128, "table layout");
  std::vector<uint32_t> g_elems_of(groups.size(), 0), g_tiles_of(groups.size(), 0);
  for (size_t g = 0; g < groups.size(); g++) {
    const std::vector<int> &G = groups[g];
    const size_t n = G.size();
    if (n == 1) continue;
    DocEntry *he = reinterpret_cast<DocEntry *>(c->h_doctab + off[g]);
    const size_t maps_at = off[g] + ((n * sizeof(DocEntry) + 127) & ~size_t(127));
    CUtensorMap *hm = reinterpret_cast<CUtensorMap *>(c->h_doctab + maps_at);
    const CUtensorMap *dm = reinterpret_cast<const CUtensorMap *>(c->d_doctab + maps_at);
    uint32_t elems = 0, tiles = 0;
    for (size_t k = 0; k < n; k++) {
      const PendingCall &pc = calls[size_t(G[k])];
      bool tma = false;
      make_tensor_map(c, &hm[k], pc.d_buf, pc.len, &tma);
      DocEntry &e = he[k];
      e.buf = pc.d_buf;
      e.idx_out = pc.d_idx;
      e.carry_out = c->d_carry + pc.carry_slot;
      e.carry_out_host = c->h_carry + pc.carry_slot;
      e.flags = c->d_flags + 1 + pc.carry_slot;
      e.tmap = tma ? static_cast<const void *>(dm + k) : nullptr;
      e.len = uint32_t(pc.len);
      e.scan_end = uint32_t(pc.len);
      e.first_elem = elems;
      e.nelem = uint32_t(elems_of(pc));
      elems += e.nelem;
      tiles += tiles_of(pc.len);
    }
    g_elems_of[g] = elems;
    g_tiles_of[g] = tiles;
  }
  if (off.back() > 0 && !ok(c, cudaMemcpyAsync(c->d_doctab, c->h_doctab, off.back(), cudaMemcpyHostToDevice, s), "H2D doc tables")) return SJB200_UNEXPECTED_ERROR;
  // early[g]: no input byte of group g lies in an index array of group g - 1, so its scan may read before that one is done
  // (the groups' carries and flags words are distinct slots of the context, no input of a caller)
  std::vector<char> early(groups.size(), 1);
  for (size_t g = 1; g < groups.size(); g++)
    for (int i : groups[g])
      for (int j : groups[g - 1])
        if (ranges_overlap(calls[size_t(i)].d_buf, calls[size_t(i)].len, calls[size_t(j)].d_idx, out_bytes(calls[size_t(j)]))) early[g] = 0;
  unsigned long long *stamps = nullptr;
  c->stamps_used = 0;
  if (c->opt_launch_stamps) {
    if (c->stamps_cap < groups.size()) {
      cudaFree(c->d_stamps); c->d_stamps = nullptr; c->stamps_cap = 0;
      if (!dev_alloc(c, &c->d_stamps, 2 * groups.size(), "cudaMalloc(stamps)")) return SJB200_MEMALLOC;
      c->stamps_cap = groups.size();
    }
    if (!ok(c, cudaMemsetAsync(c->d_stamps, 0, 16 * groups.size(), s), "memset stamps")) return SJB200_UNEXPECTED_ERROR;
    stamps = c->d_stamps;
    c->stamps_used = groups.size();
  }
  cudaEvent_t e1 = time_begin(c, s);
  uint32_t timed_docs = 0;
  bool chained = false;  // the last operation on s is this call's previous multi-document scan launch
  int parity = 0;
  for (size_t g = 0; g < groups.size(); g++) {
    const std::vector<int> &G = groups[g];
    if (G.size() == 1) {
      PendingCall &pc = calls[size_t(G[0])];
      CUtensorMap map;
      bool tma = false;
      make_tensor_map(c, &map, pc.d_buf, pc.len, &tma);
      if (!enqueue_scan(c, kIndex, &map, tma, pc.d_buf, pc.len, 0, tiles_of(pc.len), true, 0x20202020u, pc.d_idx, nullptr, -1, s, pc.carry_slot, true,
                        nullptr, c->h_carry + pc.carry_slot, nullptr, false)) {
        pc.early_error = SJB200_UNEXPECTED_ERROR;
      } else {
        timed_docs++;
        stage1_stream_epilogue(c, pc);
      }
      chained = false;
      continue;
    }
    const size_t n = G.size();
    ScanParams p;
    memset(&p, 0, sizeof(p));
    p.prev_word = 0x20202020u;
    p.check_eof = 1;
    p.write_sentinels = 1;
    p.ntiles = g_tiles_of[g];
    p.docs = reinterpret_cast<const DocEntry *>(c->d_doctab + off[g]);
    p.ndocs = uint32_t(n);
    p.early_input = early[g] ? 1u : 0u;
    p.stamps = stamps ? stamps + 2 * g : nullptr;
    bool wiped = false;
    bool good = next_epoch(c, s, &p.epoch, &wiped);
    const bool pdl = good && chained && !wiped && c->opt_pdl;
    parity = pdl ? parity ^ 1 : 0;
    p.flags = launch_flags(c, parity);
    p.count_desc = launch_desc(c, parity);
    p.ticket = launch_ticket(c, parity);
    if (good) {
      CUtensorMap unused;
      memset(&unused, 0, sizeof(unused));
      good = ok(c, launch_scan4(&unused, p, grid_for(c, g_elems_of[g]), 0, s, pdl), "launch scan4 (documents)");
      c->launches += good ? 1 : 0;
      timed_docs += good ? uint32_t(n) : 0u;
    }
    bool epilogue = false;
    for (size_t k = 0; k < n; k++) {
      PendingCall &pc = calls[size_t(G[k])];
      if (good) epilogue = stage1_stream_epilogue(c, pc) || epilogue;
      else pc.early_error = SJB200_UNEXPECTED_ERROR;
    }
    chained = good && !epilogue;
  }
  time_end(c, s, e1, timed_docs > 0, timed_docs);
  return SJB200_SUCCESS;
}
}  // namespace

// Many documents in one call (NDJSON rows, a corpus): consecutive documents share a scan launch where their memory
// allows it (enqueue_doc_groups), the launches are queued back to back on the stream, the host waits once, then
// completes each document's finish() logic.  docs[i].error receives the error_code.
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
      stage1_prepare(c, calls[size_t(i)], d.d_buf, d.len, mode, d.d_idx, s, 1 + i, tails ? tails + 4 * size_t(i) : nullptr);
    }
    const int rc = enqueue_doc_groups(c, calls, s);
    if (rc != SJB200_SUCCESS) return rc;
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
  return sjb200_document_table_shard_dev(c, d_buf, d_idx, n, 1, d_table, capacity, ndocs_out, stream);
}

// the same for one shard of a sharded stream pass: whether structural 0 starts a document came from the pass's fold
extern "C" int sjb200_document_table_shard_dev(sjb200_ctx *c, const uint8_t *d_buf, const uint32_t *d_idx, uint32_t n, int first_starts_document,
                                               sjb200_doc_boundary *d_table, uint32_t capacity, uint32_t *ndocs_out, void *stream) {
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
  if (!ok(c, launch_doc_table(d_buf, d_idx, n, first_starts_document != 0, c->d_doc_scratch, reinterpret_cast<sjb200_doc_boundary_t *>(d_table), capacity,
                              c->d_ndocs, s), "doc table") ||
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
  make_tensor_map(c, &map, d_buf, len, &tma);
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
  make_tensor_map(c, &map, d_buf, len, &tma);
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
  make_tensor_map(c, &map, c->d_in, len, &tma);
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
  uint32_t *alias = mapped_alias(c, idx_out);
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
  make_tensor_map(c, &map, d_buf, len, &tma);
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
  make_tensor_map(c, &map, d_buf, len, &tma);
  if (!enqueue_scan(c, kIndex, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, d_idx, nullptr, -1, s, 1, false,
                    static_cast<Carry *>(d_result)))
    return SJB200_UNEXPECTED_ERROR;
  return SJB200_SUCCESS;
}

// =============================================================================== sharded scan with the exchange fused in
// One object per rank.  The exchange window lives in device memory; peers map it through CUDA IPC (one process per GPU,
// the torch.distributed / MPI layout) or directly (several contexts in one process).  A pass = every rank scans its
// shard with the speculated state 0; the scan kernel's last CTA stores the 16-byte record {count, state, transducer,
// flags, kind} into every rank's window over NVLink -- no collective launch.  finish() reads the local window, folds the
// true incoming state and base, and -- only when somebody's speculation was wrong -- re-scans and runs a second round.
// A pass is stage 1 (plain, stream or delimited), minify, validate_utf8 or stage-2-lite (its kind; the tokens pass's record
// comes from tile_scan_kernel, sjb200_tape.cu); passes of all kinds share the window and may be in flight
// together, up to kXchgSteps / 2 per rank (enqueue ... enqueue, finish ... finish), as long as every rank enqueues the
// same sequence of kinds.
struct sjb200_comm {
  sjb200_ctx *ctx = nullptr;
  int rank = 0, nranks = 1;
  unsigned long long *window = nullptr;            // [kXchgSteps][2 rounds][kMaxRanks][2], then the summaries (sjb200_params.h)
  unsigned long long *peer[kMaxRanks] = {};        // peer[r] = rank r's window as seen from this device
  bool opened[kMaxRanks] = {};                     // mapped through cudaIpcOpenMemHandle (to be closed)
  bool connected = false;
  unsigned long long *h_rec = nullptr;             // pinned [kMaxRanks][kDelimWords]: records ([r][0..1]), summaries or delimited blocks
  uint32_t *h_tot = nullptr;                       // pinned [4]: a delimited pass's filter totals
  uint32_t *d_scratch = nullptr;                   // a delimited pass's filter scratch (delim_scratch_words)
  size_t scratch_words = 0;
  Carry *d_result = nullptr;                       // [kXchgSteps] the launches' own result blocks
  // tokens passes, by the slot of their pass (a pass in flight keeps its own): totals, tile scratch (grow-only)
  TokenTotals *d_tok_tot = nullptr;
  void *d_tok_scratch[kXchgSteps] = {};
  size_t tok_scratch_bytes[kXchgSteps] = {};
  cudaStream_t poll_stream = nullptr;
  cudaEvent_t done[kXchgSteps] = {};
  struct Step { const uint8_t *d_buf; size_t len; uint32_t *d_idx; uint8_t *d_dst; cudaStream_t stream; uint32_t seq; int last; int kind; int mode; } steps[kXchgSteps];
  uint32_t head = 0, tail = 0;                     // passes enqueued / finished
  long poll_timeout_ms = 20000;
};

namespace {
constexpr size_t kWindowWords = kXchgWindowWords;
uint32_t window_slot(uint32_t seq, int round) { return (seq % uint32_t(kXchgSteps)) * 2u + uint32_t(round); }

// wait (host polling, bounded) until every rank's record of (seq, round) is in the local window; records -> comm->h_rec.
// round 2: the summaries of a streaming pass (kSumWords words per rank, each tagged with seq).  round 3: words
// [first, first + nwords) of every rank's delimited block (h_rec[r * kDelimWords + k], the whole blocks are copied).
int comm_collect(sjb200_comm *m, uint32_t seq, int round, int first = 0, int nwords = 0) {
  sjb200_ctx *c = m->ctx;
  const bool sums = (round == 2), delim = (round == 3);
  const unsigned long long *src = delim  ? m->window + xchg_delim_at(seq, 0)
                                  : sums ? m->window + xchg_summary_at(seq, 0)
                                         : m->window + size_t(window_slot(seq, round)) * kMaxRanks * 2;
  const size_t words = delim ? size_t(kDelimWords) : sums ? size_t(kSumWords) : 2;
  const auto t0 = std::chrono::steady_clock::now();
  for (;;) {
    if (!ok(c, cudaMemcpyAsync(m->h_rec, src, size_t(m->nranks) * words * 8, cudaMemcpyDeviceToHost, m->poll_stream), "D2H window") ||
        !ok(c, cudaStreamSynchronize(m->poll_stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->xchg_polls++;
    bool all = true;
    for (int r = 0; r < m->nranks; r++) {
      if (delim) {
        for (int k = first; k < first + nwords; k++) all = all && uint32_t(m->h_rec[size_t(r) * kDelimWords + k] >> 32) == seq;
        continue;
      }
      if (!sums) { all = all && xchg_complete(m->h_rec[2 * r], m->h_rec[2 * r + 1], seq); continue; }
      for (int k = 0; k < kSumWords; k++) all = all && uint32_t(m->h_rec[size_t(r) * kSumWords + k] >> 32) == seq;
    }
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
              ok(c, cudaMallocHost(&hp, kMaxRanks * kDelimWords * 8 + 16), "cudaMallocHost") &&
              ok(c, cudaStreamCreateWithFlags(&m->poll_stream, cudaStreamNonBlocking), "stream");
  m->h_rec = static_cast<unsigned long long *>(hp);
  if (hp) m->h_tot = reinterpret_cast<uint32_t *>(m->h_rec + kMaxRanks * kDelimWords);
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
  cudaFree(m->window); cudaFree(m->d_result); cudaFree(m->d_scratch); cudaFree(m->d_tok_tot);
  for (void *p : m->d_tok_scratch) cudaFree(p);
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

namespace {
// Enqueue one pass of `kind` (kIndex: d_idx, kMinify: d_dst, kUtf8: neither).  The launch's record lands in every rank's
// window; m->done[slot] marks the end of the launch on `stream`.
int sharded_enqueue(sjb200_comm *m, int kind, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx, uint8_t *d_dst, void *stream,
                    int mode = SJB200_REGULAR) {
  const bool idx_kind = (kind == kIndex || kind == kStream || kind == kDelim);
  if (!m || !m->connected || !d_shard || len == 0 || len > kMaxBytes || (idx_kind && !d_idx) || (kind == kMinify && !d_dst))
    return SJB200_UNEXPECTED_ERROR;
  if (kind == kStream && (mode < SJB200_REGULAR || mode > SJB200_STREAMING_FINAL)) return SJB200_UNEXPECTED_ERROR;
  if (kind == kDelim && (mode < SJB200_JSON_SEQUENCE_PARTIAL || mode > SJB200_COMMA_DELIMITED_FINAL)) return SJB200_UNEXPECTED_ERROR;
  if (m->head - m->tail >= uint32_t(kXchgSteps / 2)) return SJB200_CAPACITY;  // too many passes in flight: finish some first
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const auto t_enq = std::chrono::steady_clock::now();
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if ((kind == kStream || kind == kDelim) && last_shard && mode != SJB200_REGULAR) {  // the partial UTF-8 trim of the stream's end (json_structural_indexer.h L198-204)
    const size_t k = std::min<size_t>(3, len);
    if (!ok(c, cudaMemcpyAsync(c->h_small, d_shard + len - k, k, cudaMemcpyDeviceToHost, s), "D2H tail") || !ok(c, cudaStreamSynchronize(s), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    len = trim_partial_utf8_tail(c->h_small, k, len);
  }
  const int scan_kind = idx_kind ? kIndex : kind;  // stream and delimited passes scan like stage 1; only their records' kind differs
  if (scan_kind != kUtf8 && len && !ensure_desc(c, len)) return SJB200_MEMALLOC;  // (scan4's look-back descriptors)
  const uint32_t seq = m->head + 1;  // tags start at 1: a zeroed window never matches
  XchgTarget x;
  for (int r = 0; r < kMaxRanks; r++) x.peer[r] = m->peer[r];
  x.nranks = uint32_t(m->nranks); x.rank = uint32_t(m->rank); x.slot = window_slot(seq, 0); x.seq = seq; x.kind = uint32_t(kind);
  const uint32_t i = m->head % uint32_t(kXchgSteps);
  sjb200_comm::Step &st = m->steps[i];
  st.d_buf = d_shard; st.len = len; st.d_idx = d_idx; st.d_dst = d_dst; st.stream = s; st.seq = seq; st.last = last_shard; st.kind = kind; st.mode = mode;
  bool good;
  if (len == 0) {  // a last shard that trims to nothing: no scan; its record {count 0, escape passed through, no flags}
    ScanParams p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < kMaxRanks; r++) p.xchg_peer[r] = x.peer[r];
    p.xchg_nranks = x.nranks; p.xchg_rank = x.rank; p.xchg_slot = x.slot; p.xchg_seq = seq;
    good = ok(c, launch_xchg_post(p, xchg_word0(seq, 0), xchg_word1(seq, 0, 0x8u, 0, kind), s), "xchg post");
    c->launches += good ? 1 : 0;
  } else {
    CUtensorMap map;
    bool tma = false;
    make_tensor_map(c, &map, d_shard, len, &tma);
    good = enqueue_scan(c, scan_kind, &map, tma, d_shard, len, 0, tiles_of(len), true, 0x20202020u, d_idx, d_dst, -1, s, 1, false, m->d_result + i, nullptr, &x);
  }
  if (!good || !ok(c, cudaEventRecord(m->done[i], s), "event record"))
    return SJB200_UNEXPECTED_ERROR;
  m->head++;
  c->xchg_enqueue_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enq).count();
  return SJB200_SUCCESS;
}

// the minify counterpart of sjb200_stage1_shard_dev, for the second round: minify the shard again from its true incoming
// state (carry slot 0 = that state and count 0, so the kept bytes start at d_dst[0])
int minify_shard_from(sjb200_ctx *c, const uint8_t *d_buf, size_t len, uint32_t state_in, uint8_t *d_dst, cudaStream_t s, uint64_t *count, uint32_t *flags) {
  if (!ensure_desc(c, len)) return SJB200_MEMALLOC;
  CUtensorMap map;
  bool tma = false;
  make_tensor_map(c, &map, d_buf, len, &tma);
  c->h_carry[0].count = 0; c->h_carry[0].state = state_in & 7u; c->h_carry[0].ttable = 0;
  c->h_carry[0].flags = 0; c->h_carry[0].reserved = 0;
  if (!ok(c, cudaMemcpyAsync(c->d_carry, c->h_carry, sizeof(Carry), cudaMemcpyHostToDevice, s), "H2D carry") ||
      !enqueue_scan(c, kMinify, &map, tma, d_buf, len, 0, tiles_of(len), true, 0x20202020u, nullptr, d_dst, 0, s) ||
      !fetch_result(c, s) || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  *count = c->h_carry[1].count;
  *flags = c->h_carry[1].flags & kFlagInternal;  // as in the kernel's record: the only flag that means something to minify
  return *flags ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
}

// Complete the oldest pass in flight, which must be of `kind`: the one body of the three sharded finishes.
int sharded_finish(sjb200_comm *m, int kind, sjb200_sharded_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  memset(out, 0, sizeof(*out));
  const uint32_t slot_i = m->tail % uint32_t(kXchgSteps);
  const sjb200_comm::Step st = m->steps[slot_i];
  if (st.kind != kind) {  // (the pass stays in flight: the caller can still finish it with the right call)
    c->last_error = "sharded finish: the oldest pass in flight is of another kind";
    return SJB200_UNEXPECTED_ERROR;
  }
  m->tail++;
  const auto t_ev = std::chrono::steady_clock::now();
  if (!ok(c, cudaEventSynchronize(m->done[slot_i]), "event sync")) return SJB200_UNEXPECTED_ERROR;  // own scan (and its stores) done
  c->xchg_evsync_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_ev).count();
  int rc = comm_collect(m, st.seq, 0);
  if (rc != SJB200_SUCCESS) return rc;
  for (int r = 0; r < m->nranks; r++)
    if (xchg_kind(m->h_rec[2 * r + 1]) != kind) {  // never fold one kind's counts into another's base
      c->last_error = "sharded pass " + std::to_string(st.seq) + ": rank " + std::to_string(r) + " published a pass of another kind (every rank must enqueue the same sequence of kinds)";
      return SJB200_UNEXPECTED_ERROR;
    }
  // A speculation (state 0) is wrong when the true incoming state changes what the scan keeps: for stage 1 any bit does
  // (bit 2 decides whether a scalar starts), for minify only escape and in-string do.  validate_utf8 records carry
  // transducer 0, so its states are all 0.
  const uint32_t matters = (kind == kMinify) ? 3u : 7u;
  uint32_t tt[kMaxRanks], flags_all = 0;
  bool any_wrong = false;
  uint32_t state = 0, my_state = 0;
  for (int r = 0; r < m->nranks; r++) {
    tt[r] = uint32_t(m->h_rec[2 * r + 1] >> 8) & 0x3Fu;
    if (r == m->rank) my_state = state;
    if ((state & matters) != 0) any_wrong = true;
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
    if ((my_state & matters) != 0 && st.len > 0) {  // (a stream's last shard that trimmed to nothing has nothing to scan)
      if (kind != kMinify) {
        sjb200_shard_result sr;
        rc = sjb200_stage1_shard_dev(c, st.d_buf, st.len, my_state, st.last, st.d_idx, &sr, st.stream);
        my_count = sr.count;
        my_flags = sr.flags;
      } else {
        rc = minify_shard_from(c, st.d_buf, st.len, my_state, st.d_dst, st.stream, &my_count, &my_flags);
      }
      if (rc != SJB200_SUCCESS) return rc;
      out->rescanned = 1;
    }
    ScanParams p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < kMaxRanks; r++) p.xchg_peer[r] = m->peer[r];
    p.xchg_nranks = uint32_t(m->nranks); p.xchg_rank = uint32_t(m->rank); p.xchg_slot = window_slot(st.seq, 1); p.xchg_seq = st.seq;
    if (!ok(c, launch_xchg_post(p, xchg_word0(st.seq, my_count), xchg_word1(st.seq, out->state_out, tt[m->rank], my_flags, kind), st.stream), "xchg post") ||
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
  if ((my_flags | flags_all) & kFlagInternal) return SJB200_UNEXPECTED_ERROR;
  if (kind == kMinify && ((state >> 1) & 1u)) return SJB200_UNCLOSED_STRING;  // the document ends inside a string: json_minifier.h L42-47
  return SJB200_SUCCESS;
}

// the kSumWords words of stream_summary_kernel (sjb200_params.h) -> the fold's summary of `count` structurals
void decode_summary(const unsigned long long *w, uint64_t count, sjb200_stream_summary *out) {
  sjb200_stream_summary &s = *out;
  s.count = count;
  s.len = uint32_t(w[0]); s.first_byte = uint32_t(w[1]); s.last_byte = uint32_t(w[2]);
  s.start_index = uint32_t(w[3]); s.start_byte = uint32_t(w[4]);
  s.net_obj = int32_t(uint32_t(w[5])); s.net_arr = int32_t(uint32_t(w[6]));
  s.role_first = uint32_t(w[7]) & 7u; s.role_last = (uint32_t(w[7]) >> 3) & 7u; s.has_start = (uint32_t(w[7]) >> 6) & 1u;
}

// Complete the oldest pass in flight, a stream pass: the scan's fold (sharded_finish), then the summary round and the
// host fold of the whole stream's finish() (sjb200_stream_fold), then this rank's sentinels and rewrites.
int sharded_stream_finish(sjb200_comm *m, sjb200_sharded_stream_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  memset(out, 0, sizeof(*out));
  const sjb200_comm::Step st = m->steps[m->tail % uint32_t(kXchgSteps)];
  int rc = sharded_finish(m, kStream, &out->shard);
  if (rc != SJB200_SUCCESS) return rc;  // (an internal error is seen by every rank alike: nobody runs the summary round)
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  // h_rec holds every rank's last record: the counts after the second round
  uint64_t counts[kMaxRanks];
  int holder = -1;  // the rank that holds the stream's last structural
  for (int r = 0; r < m->nranks; r++) {
    counts[r] = xchg_count(m->h_rec[2 * r]);
    if (counts[r]) holder = r;
  }
  const bool unclosed = (out->shard.final_state >> 1) & 1u;
  const uint64_t my_count = counts[m->rank];
  const uint64_t kept = my_count - ((st.mode != SJB200_REGULAR && unclosed && holder == m->rank) ? 1 : 0);
  ScanParams x;
  memset(&x, 0, sizeof(x));
  for (int r = 0; r < kMaxRanks; r++) x.xchg_peer[r] = m->peer[r];
  x.xchg_nranks = uint32_t(m->nranks); x.xchg_rank = uint32_t(m->rank); x.xchg_seq = st.seq;
  if (!ok(c, launch_stream_summary(st.d_buf, st.d_idx, uint32_t(my_count), uint32_t(kept), uint32_t(st.len), st.mode != SJB200_REGULAR, x,
                                   xchg_summary_at(st.seq, uint32_t(m->rank)), m->poll_stream),
          "stream summary"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches++;
  rc = comm_collect(m, st.seq, 2);
  if (rc != SJB200_SUCCESS) return rc;
  sjb200_stream_summary sums[kMaxRanks];
  for (int r = 0; r < m->nranks; r++) decode_summary(m->h_rec + size_t(r) * kSumWords, counts[r], &sums[r]);
  sjb200_stream_fold_result res;
  sjb200_stream_rank ranks[kMaxRanks];
  const int err = sjb200_stream_fold(st.mode, m->nranks, out->shard.final_state, out->shard.flags_all, sums, &res, ranks);
  const sjb200_stream_rank &me = ranks[m->rank];
  out->n = res.n;
  out->kept = me.kept;
  out->bytes_before = me.bytes_before;
  out->total_bytes = res.total_bytes;
  out->first_starts_document = me.first_starts_document;
  // the stream's sentinels (json_structural_indexer.h L284-286) go behind the last rank's count, then the final fix-up
  const bool sentinels = res.n_written && st.last;
  if (sentinels || me.nrewrites) {
    if ((sentinels && !ok(c, launch_write_sentinels(st.d_idx, uint32_t(my_count), uint32_t(st.len), uint32_t(st.len), 0, m->poll_stream), "sentinels")) ||
        (me.nrewrites && !ok(c, launch_store_words(st.d_idx, me.nrewrites, me.rewrite_pos[0], me.rewrite_val[0], me.rewrite_pos[1], me.rewrite_val[1],
                                                  m->poll_stream), "rewrite")) ||
        !ok(c, cudaStreamSynchronize(m->poll_stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->launches += (sentinels ? 1 : 0) + (me.nrewrites ? 1 : 0);
  }
  return err;
}
}  // namespace

// Complete the oldest pass in flight, a delimited pass (modes 3..6): the scan's fold (sharded_finish), then three rounds,
// each a small kernel storing tagged words into every rank's window and a comm_collect (DESIGN.md section 5):
//   carry   every rank's length and the bracket net (comma) or "ends inside a separator run" / "whitespace / RS only"
//           (RS) -> this rank's depth_in / run_in;
//   filter  the filter of sjb200_docs.cu with that carry, into the scratch, then its totals and the walks of
//           find_next_document_index over the filtered entries -> sjb200_delimited_fold;
//   tail    the holders of the words n, n+1, n+2 publish them (skipped when the fold knows all three); then the
//           filtered entries go back into d_idx.
namespace {
int sharded_delimited_finish(sjb200_comm *m, sjb200_sharded_delimited_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  memset(out, 0, sizeof(*out));
  const sjb200_comm::Step st = m->steps[m->tail % uint32_t(kXchgSteps)];
  int rc = sharded_finish(m, kDelim, &out->stream.shard);
  if (rc != SJB200_SUCCESS) return rc;  // (an internal error is seen by every rank alike: nobody runs the extra rounds)
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const int me = m->rank;
  uint64_t counts[kMaxRanks];
  int holder = -1;  // the rank that holds the stream's last structural
  for (int r = 0; r < m->nranks; r++) {
    counts[r] = xchg_count(m->h_rec[2 * r]);
    if (counts[r]) holder = r;
  }
  const bool unclosed = (out->stream.shard.final_state >> 1) & 1u;
  const bool comma = (st.mode == SJB200_COMMA_DELIMITED_PARTIAL || st.mode == SJB200_COMMA_DELIMITED_FINAL);
  const bool walk_below = (st.mode == SJB200_COMMA_DELIMITED_PARTIAL);
  // the structurals this shard's filter considers: less the stream's last one when it ends inside a string
  const uint32_t n = uint32_t(counts[me]) - ((unclosed && holder == me) ? 1u : 0u);
  const uint32_t len = uint32_t(st.len);
  const size_t need = delim_scratch_words(n);
  if (m->scratch_words < need) {
    cudaFree(m->d_scratch); m->d_scratch = nullptr; m->scratch_words = 0;
    if (!dev_alloc(c, &m->d_scratch, need, "cudaMalloc(delimited scratch)")) return SJB200_MEMALLOC;
    m->scratch_words = need;
  }
  ScanParams x;
  memset(&x, 0, sizeof(x));
  for (int r = 0; r < kMaxRanks; r++) x.xchg_peer[r] = m->peer[r];
  x.xchg_nranks = uint32_t(m->nranks); x.xchg_rank = uint32_t(me); x.xchg_seq = st.seq;
  const size_t at = xchg_delim_at(st.seq, uint32_t(me));
  cudaStream_t s = m->poll_stream;
  // carry round
  if (!ok(c, launch_delim_carry(st.d_buf, st.d_idx, n, len, comma, m->d_scratch, x, at + kDelimCarryAt, s), "delimited carry")) return SJB200_UNEXPECTED_ERROR;
  c->launches++;
  if ((rc = comm_collect(m, st.seq, 3, kDelimCarryAt, kDelimCarryWords)) != SJB200_SUCCESS) return rc;
  uint32_t lens[kMaxRanks];
  int depth = 0, depth_in = 0;
  bool run = false, run_in = false;  // run: the bytes from an RS entry of an earlier shard up to here are whitespace / RS
  for (int r = 0; r < m->nranks; r++) {
    const unsigned long long *w = m->h_rec + size_t(r) * kDelimWords + kDelimCarryAt;
    lens[r] = uint32_t(w[0]);
    if (r == me) { depth_in = depth; run_in = run; }
    if (comma) depth += int32_t(uint32_t(w[1]));
    else run = uint32_t(w[1]) != 0 || (run && uint32_t(w[2]) != 0);
  }
  // filter round
  if (!ok(c, launch_delim_filter(st.d_buf, len, st.d_idx, n, comma, depth_in, run_in, m->d_scratch, m->h_tot, s), "delimited filter") ||
      !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  const uint32_t filtered = m->h_tot[0], below = m->h_tot[3];
  const uint32_t *dst = delim_filtered(m->d_scratch);
  if (!ok(c, launch_stream_summary(st.d_buf, dst, filtered, filtered, len, 1, x, at + kDelimWalkAt, s), "delimited walk") ||
      (walk_below && !ok(c, launch_stream_summary(st.d_buf, dst, below, below, len, 1, x, at + kDelimWalkBelowAt, s), "delimited walk")) ||
      !ok(c, launch_delim_publish_totals(m->d_scratch, n, x, at + kDelimTotalsAt, s), "delimited totals"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += 6 + (walk_below ? 1 : 0);
  const int upto = walk_below ? kDelimTailAt : kDelimWalkBelowAt;
  if ((rc = comm_collect(m, st.seq, 3, kDelimTotalsAt, upto - kDelimTotalsAt)) != SJB200_SUCCESS) return rc;
  sjb200_delimited_summary sums[kMaxRanks];
  memset(sums, 0, sizeof(sums));
  for (int r = 0; r < m->nranks; r++) {
    const unsigned long long *w = m->h_rec + size_t(r) * kDelimWords;
    sjb200_delimited_summary &d = sums[r];
    d.count = counts[r]; d.len = lens[r];
    d.filtered = uint32_t(w[kDelimTotalsAt]); d.seps = uint32_t(w[kDelimTotalsAt + 1]);
    d.last_sep = uint32_t(w[kDelimTotalsAt + 2]); d.below = uint32_t(w[kDelimTotalsAt + 3]);
    decode_summary(w + kDelimWalkAt, d.filtered, &d.walk);
    if (walk_below) decode_summary(w + kDelimWalkBelowAt, d.below, &d.walk_below);
  }
  sjb200_delimited_fold_result res;
  sjb200_delimited_rank ranks[kMaxRanks];
  const int err = sjb200_delimited_fold(st.mode, m->nranks, out->stream.shard.final_state, out->stream.shard.flags_all, sums, &res, ranks);
  out->stream.n = res.n;
  out->stream.kept = ranks[me].kept;
  out->stream.bytes_before = ranks[me].bytes_before;
  out->stream.total_bytes = res.total_bytes;
  out->stream.first_starts_document = ranks[me].first_starts_document;
  out->filtered = filtered;
  out->filtered_before = ranks[me].filtered_before;
  // tail round
  DelimTail t;
  memset(&t, 0, sizeof(t));
  t.add = uint32_t(ranks[me].bytes_before);
  bool publish = false;
  for (int k = 0; k < 3; k++) {
    if (res.tail_rank[k] < 0) continue;
    publish = true;
    if (res.tail_rank[k] == me) { t.src[k] = res.tail_filtered[k] ? 1 : 2; t.pos[k] = res.tail_pos[k]; }
  }
  if (!ok(c, launch_delim_tail(m->d_scratch, n, st.d_idx, t, publish, x, at + kDelimTailAt, s), "delimited tail") ||
      !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += publish ? 2 : 1;
  if (publish && (rc = comm_collect(m, st.seq, 3, kDelimTailAt, 3)) != SJB200_SUCCESS) return rc;
  for (int k = 0; k < 3; k++)
    out->tail[k] = res.tail_rank[k] < 0 ? res.tail_val[k] : uint32_t(m->h_rec[size_t(res.tail_rank[k]) * kDelimWords + kDelimTailAt + k]);
  return err;
}
}  // namespace

extern "C" int sjb200_stage1_sharded_stream_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                                    void *stream) {
  return sharded_enqueue(m, kStream, d_shard, len, last_shard, d_idx, nullptr, stream, mode);
}

extern "C" int sjb200_stage1_sharded_stream_finish(sjb200_comm *m, sjb200_sharded_stream_result *out) { return sharded_stream_finish(m, out); }

extern "C" int sjb200_stage1_sharded_stream(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                            sjb200_sharded_stream_result *out, void *stream) {
  int rc = sjb200_stage1_sharded_stream_enqueue(m, d_shard, len, last_shard, mode, d_idx, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_stage1_sharded_stream_finish(m, out);
}

namespace {
enum : uint32_t { kRoleValue = 0, kRoleSep, kRoleOpenObj, kRoleCloseObj, kRoleOpenArr, kRoleCloseArr };  // as in sjb200_docs.cu
bool starts_document(uint32_t cur, uint32_t before) {  // find_next_document_index.h L60-88
  if (cur == kRoleSep || cur == kRoleCloseObj || cur == kRoleCloseArr) return false;
  return !(before == kRoleOpenObj || before == kRoleOpenArr || before == kRoleSep);
}
}  // namespace

// The fold of the summaries into the whole stream's finish() (json_structural_indexer.h L249-343, L395-396).  T = all
// structurals, n0 = T less the stream's last one when it ends inside a string (streaming modes).  The last document start
// g of [0, n0) is the last internal start of the last shard that has one, unless the first structural of a later shard
// starts a document across its cut; the brackets from g on are that shard's nets after its start plus the later shards'
// nets.  Then m = n0 when they balance, else g (0 without any start), as find_next_document_index.
extern "C" int sjb200_stream_fold(int mode, int nranks, uint32_t final_state, uint32_t flags_all, const sjb200_stream_summary *sums,
                                  sjb200_stream_fold_result *res, sjb200_stream_rank *ranks) {
  if (!res || !ranks || !sums || nranks < 1 || nranks > kMaxRanks || mode < SJB200_REGULAR || mode > SJB200_STREAMING_FINAL) return SJB200_UNEXPECTED_ERROR;
  memset(res, 0, sizeof(*res));
  memset(ranks, 0, sizeof(*ranks) * size_t(nranks));
  uint64_t base[kMaxRanks], off = 0, T = 0;
  int holder = -1;
  for (int r = 0; r < nranks; r++) {
    ranks[r].bytes_before = off;
    off += sums[r].len;
    base[r] = T;
    T += sums[r].count;
    if (sums[r].count) holder = r;
  }
  const uint64_t L = off;
  res->total_bytes = L;
  const bool streaming = mode != SJB200_REGULAR, unclosed = (final_state >> 1) & 1u;
  auto done = [&](int err) {
    res->error = err;
    for (int r = 0; r < nranks && res->n_written; r++) {
      const uint64_t k = res->n > base[r] ? res->n - base[r] : 0;
      ranks[r].kept = std::min<uint64_t>(k, sums[r].count);
    }
    for (int r = 0, prev = -1; r < nranks; r++) {  // prev: the last earlier shard with kept structurals
      if (ranks[r].kept == 0) continue;
      ranks[r].first_starts_document = (prev < 0) ? 1u : uint32_t(starts_document(sums[r].role_first, sums[prev].role_last));
      prev = r;
    }
    return err;
  };
  if (flags_all & kFlagInternal) return done(SJB200_UNEXPECTED_ERROR);
  if (streaming && L == 0) return done(SJB200_UTF8_ERROR);           // L198-204: nothing left after the trim
  if (!streaming && unclosed) return done(SJB200_UNCLOSED_STRING);   // L255-259
  if (flags_all & kFlagCtl) return done(SJB200_UNESCAPED_CHARS);    // L261-263
  res->n_written = 1;
  res->n = T;
  if (T == 0) return done(SJB200_EMPTY);                             // L289-291
  const bool utf8 = (flags_all & kFlagUtf8) != 0;
  if (!streaming) return done(utf8 ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
  const uint64_t n0 = T - (unclosed ? 1 : 0);
  if (mode == SJB200_STREAMING_PARTIAL && unclosed && n0 == 0) { res->n = 0; return done(SJB200_CAPACITY); }  // L298-302
  // the last document start g < n0 and the bracket balance of [g, n0); gv = global byte of structural g
  uint64_t g = 0, gv = 0;
  bool found = false;
  int64_t nobj = 0, narr = 0;
  for (int r = nranks - 1; r >= 0 && !found; r--) {
    const uint64_t kp = sums[r].count - ((unclosed && r == holder) ? 1 : 0);
    if (kp == 0) continue;
    nobj += sums[r].net_obj;
    narr += sums[r].net_arr;
    if (sums[r].has_start) {
      found = true; g = base[r] + sums[r].start_index; gv = ranks[r].bytes_before + sums[r].start_byte;
    } else if (base[r] > 0) {
      int q = r - 1;
      while (q >= 0 && sums[q].count == 0) q--;
      if (q >= 0 && starts_document(sums[r].role_first, sums[q].role_last)) { found = true; g = base[r]; gv = ranks[r].bytes_before + sums[r].first_byte; }
    }
  }
  if (!found && n0 > 0) {  // the start is structural 0
    int r0 = 0;
    while (sums[r0].count == 0) r0++;
    gv = ranks[r0].bytes_before + sums[r0].first_byte;
  }
  const uint64_t m = (n0 == 0) ? 0 : ((nobj == 0 && narr == 0) ? n0 : g);
  if (mode == SJB200_STREAMING_PARTIAL) {  // L303-317
    if (m == 0) {
      const bool idx0_zero = sums[0].count > 0 && sums[0].first_byte == 0;
      if (idx0_zero) { res->n = n0; return done(SJB200_CAPACITY); }
      res->n = 0;
      return done(SJB200_EMPTY);
    }
    res->n = m;
    return done(utf8 ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
  }
  // streaming final, L329-343: word m + 1 = old word m, word m = L; the ranks that hold them store them shard-relative
  uint64_t old_m;
  if (m >= T) old_m = L;                                                            // a sentinel
  else if (m == T - 1 && unclosed) old_m = ranks[holder].bytes_before + sums[holder].last_byte;  // the dropped quote
  else old_m = gv;                                                                  // a document start
  const uint64_t pos[2] = {m, m + 1}, val[2] = {L, old_m};
  for (int k = 0; k < 2; k++) {
    int r = nranks - 1;
    uint64_t local = sums[r].count + (pos[k] - T);
    if (pos[k] < T) {
      r = 0;
      while (!(pos[k] >= base[r] && pos[k] < base[r] + sums[r].count)) r++;
      local = pos[k] - base[r];
    }
    sjb200_stream_rank &w = ranks[r];
    w.rewrite_pos[w.nrewrites] = uint32_t(local);
    w.rewrite_val[w.nrewrites] = uint32_t(val[k] - w.bytes_before);
    w.nrewrites++;
  }
  res->n = m;
  if (m == 0) return done(SJB200_EMPTY);
  return done(utf8 ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
}

extern "C" int sjb200_stage1_sharded_delimited_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                                       void *stream) {
  return sharded_enqueue(m, kDelim, d_shard, len, last_shard, d_idx, nullptr, stream, mode);
}

extern "C" int sjb200_stage1_sharded_delimited_finish(sjb200_comm *m, sjb200_sharded_delimited_result *out) { return sharded_delimited_finish(m, out); }

extern "C" int sjb200_stage1_sharded_delimited(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, int mode, uint32_t *d_idx,
                                               sjb200_sharded_delimited_result *out, void *stream) {
  int rc = sjb200_stage1_sharded_delimited_enqueue(m, d_shard, len, last_shard, mode, d_idx, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_stage1_sharded_delimited_finish(m, out);
}

// ---------------------------------------------------------------------------------------------- sharded stage-2-lite
// Enqueue one tokens pass: the launches of sjb200_tokens_dev on the shard, on the totals and tile scratch of the pass's
// own slot (passes of every kind may be in flight), with tile_scan_kernel storing the record and the summary into every
// rank's window.  A rank that cannot run its pass (device allocation) still publishes a record, with kFlagInternal, so
// that every rank's finish fails alike instead of waiting for it.
extern "C" int sjb200_tokens_sharded_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, uint32_t state_in, const uint32_t *d_idx, uint32_t n,
                                             uint8_t *d_type, uint64_t *d_payload, uint8_t *d_strbuf, size_t strbuf_capacity, void *stream) {
  if (!m || !m->connected || len > kMaxBytes || state_in > 7u || (n && (!d_shard || !d_idx || !d_type || !d_payload)) || (strbuf_capacity && !d_strbuf))
    return SJB200_UNEXPECTED_ERROR;
  if (m->head - m->tail >= uint32_t(kXchgSteps / 2)) return SJB200_CAPACITY;  // too many passes in flight: finish some first
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const auto t_enq = std::chrono::steady_clock::now();
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  const uint32_t seq = m->head + 1, i = m->head % uint32_t(kXchgSteps);
  sjb200_comm::Step &st = m->steps[i];
  st.d_buf = d_shard; st.len = len; st.d_idx = nullptr; st.d_dst = nullptr; st.stream = s; st.seq = seq; st.last = 0; st.kind = kTokens; st.mode = 0;
  TokXchg x{};
  for (int r = 0; r < kMaxRanks; r++) x.peer[r] = m->peer[r];
  x.nranks = uint32_t(m->nranks); x.rank = uint32_t(m->rank); x.slot = window_slot(seq, 0); x.seq = seq;
  x.state_in = state_in; x.n = n; x.len = len; x.capacity = strbuf_capacity;
  const size_t need = tokens_scratch_bytes(n);
  bool have = m->d_tok_tot || dev_alloc(c, &m->d_tok_tot, kXchgSteps, "cudaMalloc(token totals)");
  if (have && m->tok_scratch_bytes[i] < need) {  // (the slot's previous pass has been finished: at most kXchgSteps / 2 are in flight)
    cudaFree(m->d_tok_scratch[i]); m->d_tok_scratch[i] = nullptr; m->tok_scratch_bytes[i] = 0;
    have = ok(c, cudaMalloc(&m->d_tok_scratch[i], need), "cudaMalloc(token scratch)");
    if (have) m->tok_scratch_bytes[i] = need;
  }
  bool good;
  if (have) {
    good = ok(c, launch_tokens(d_shard, len, d_idx, n, d_type, d_payload, d_strbuf, strbuf_capacity, m->d_tok_scratch[i], m->d_tok_tot + i,
                               int(c->opt_tok_stage), s, &x), "tokens");
    c->launches += good ? (n ? 3 : 1) : 0;
  } else {
    ScanParams p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < kMaxRanks; r++) p.xchg_peer[r] = m->peer[r];
    p.xchg_nranks = x.nranks; p.xchg_rank = x.rank; p.xchg_slot = x.slot; p.xchg_seq = seq;
    good = ok(c, launch_xchg_post(p, xchg_word0(seq, 0), xchg_word1(seq, state_in, 0, kFlagInternal, kTokens), s), "xchg post");
    c->launches += good ? 1 : 0;
  }
  if (!good || !ok(c, cudaEventRecord(m->done[i], s), "event record")) return SJB200_UNEXPECTED_ERROR;
  m->head++;
  c->xchg_enqueue_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enq).count();
  return SJB200_SUCCESS;
}

// Complete the oldest pass in flight, a tokens pass: the own pass's event, the records (round 0: kind, dirty cuts, short
// and failed ranks), the summaries (round 2), then the fold of the bases and of the first error.  No second round: a
// dirty cut is refused, not re-run.
extern "C" int sjb200_tokens_sharded_finish(sjb200_comm *m, sjb200_sharded_tokens_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  memset(out, 0, sizeof(*out));
  out->error = SJB200_UNEXPECTED_ERROR;
  out->first_error_index = UINT64_MAX;
  const uint32_t slot_i = m->tail % uint32_t(kXchgSteps);
  const sjb200_comm::Step st = m->steps[slot_i];
  if (st.kind != kTokens) {  // (the pass stays in flight: the caller can still finish it with the right call)
    c->last_error = "sharded finish: the oldest pass in flight is of another kind";
    return SJB200_UNEXPECTED_ERROR;
  }
  m->tail++;
  const auto t_ev = std::chrono::steady_clock::now();
  if (!ok(c, cudaEventSynchronize(m->done[slot_i]), "event sync")) return SJB200_UNEXPECTED_ERROR;  // own launches (and their stores) done
  c->xchg_evsync_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_ev).count();
  int rc = comm_collect(m, st.seq, 0);
  if (rc != SJB200_SUCCESS) return rc;
  int failed = -1;
  for (int r = 0; r < m->nranks; r++) {
    const unsigned long long w1 = m->h_rec[2 * r + 1];
    if (xchg_kind(w1) != kTokens) {
      c->last_error = "sharded pass " + std::to_string(st.seq) + ": rank " + std::to_string(r) + " published a pass of another kind (every rank must enqueue the same sequence of kinds)";
      return SJB200_UNEXPECTED_ERROR;
    }
    const uint32_t fl = uint32_t(w1 >> 16) & 0xFFu;
    if (w1 & 7u) out->dirty_cuts |= 1u << r;
    if (fl & kTokShortFlag) out->short_ranks |= 1u << r;
    if ((fl & kFlagInternal) && failed < 0) failed = r;
  }
  if (out->dirty_cuts) {
    const int r = __builtin_ctz(out->dirty_cuts);
    c->last_error = "sharded tokens pass " + std::to_string(st.seq) + ": rank " + std::to_string(r) + " starts in state " +
                    std::to_string(m->h_rec[2 * r + 1] & 7u) + ", inside a token (tokens need cuts where the state is 0, e.g. after a line feed)";
    return SJB200_UNEXPECTED_ERROR;
  }
  if (failed >= 0) {
    if (failed != m->rank) c->last_error = "sharded tokens pass " + std::to_string(st.seq) + ": rank " + std::to_string(failed) + " could not run its pass";
    return SJB200_UNEXPECTED_ERROR;
  }
  rc = comm_collect(m, st.seq, 2);
  if (rc != SJB200_SUCCESS) return rc;
  uint64_t tokens = 0, bytes = 0, strings = 0, string_bytes = 0;
  int err = SJB200_SUCCESS;
  for (int r = 0; r < m->nranks; r++) {
    const unsigned long long *w = m->h_rec + size_t(r) * kSumWords;
    const uint64_t sb = uint64_t(uint32_t(w[5])) | (uint64_t(uint32_t(w[6])) << 32);
    const uint32_t code = uint32_t(w[4]) & 0xFFu;
    if (err == SJB200_SUCCESS && code != 0) {  // the earliest rank's first token in error
      err = int(code);
      out->first_error_index = tokens + uint32_t(w[3]);
    }
    if (r == m->rank) {
      out->tokens_before = tokens; out->bytes_before = bytes; out->strings_before = strings; out->string_base = string_bytes;
      out->n_strings = uint32_t(w[2]); out->string_bytes = sb;
    }
    tokens += uint32_t(w[1]); bytes += uint32_t(w[0]); strings += uint32_t(w[2]); string_bytes += sb;
  }
  out->total_strings = strings;
  out->total_string_bytes = string_bytes;
  if (err == SJB200_SUCCESS && out->short_ranks) err = SJB200_CAPACITY;
  out->error = err;
  return err;
}

extern "C" int sjb200_tokens_sharded(sjb200_comm *m, const uint8_t *d_shard, size_t len, uint32_t state_in, const uint32_t *d_idx, uint32_t n,
                                     uint8_t *d_type, uint64_t *d_payload, uint8_t *d_strbuf, size_t strbuf_capacity, sjb200_sharded_tokens_result *out,
                                     void *stream) {
  int rc = sjb200_tokens_sharded_enqueue(m, d_shard, len, state_in, d_idx, n, d_type, d_payload, d_strbuf, strbuf_capacity, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_tokens_sharded_finish(m, out);
}

// The fold of a delimited pass's filter round into the whole stream's finish() for modes 3..6 (json_structural_indexer.h
// L344-396 with find_next_document_index_json_sequence / filter_comma_delimited, as filter_finish_kernel runs it on one
// GPU).  The filtered entries are sorted across the ranks, so the global last separator is the last one of the last
// rank that counted any, and the entries before it are the filtered entries of the ranks before plus its `below`.
// find_next_document_index over the first k filtered entries is sjb200_stream_fold's walk over the ranks' walk
// summaries (every rank's full walk, the last rank's walk_below when k ends at its `below`).  The words after n are those
// of the array the reference's in-place filter leaves: the filtered entries, then the scan's structurals, then the
// sentinels len, len, 0.
extern "C" int sjb200_delimited_fold(int mode, int nranks, uint32_t final_state, uint32_t flags_all, const sjb200_delimited_summary *sums,
                                     sjb200_delimited_fold_result *res, sjb200_delimited_rank *ranks) {
  if (!res || !ranks || !sums || nranks < 1 || nranks > kMaxRanks || mode < SJB200_JSON_SEQUENCE_PARTIAL || mode > SJB200_COMMA_DELIMITED_FINAL)
    return SJB200_UNEXPECTED_ERROR;
  memset(res, 0, sizeof(*res));
  memset(ranks, 0, sizeof(*ranks) * size_t(nranks));
  uint64_t base[kMaxRanks], off = 0, T = 0, W = 0, seps = 0;
  int sep_rank = -1;  // the last rank that counted a separator
  for (int r = 0; r < nranks; r++) {
    ranks[r].bytes_before = off;
    ranks[r].filtered_before = W;
    off += sums[r].len;
    base[r] = T;
    T += sums[r].count;
    W += sums[r].filtered;
    seps += sums[r].seps;
    if (sums[r].seps) sep_rank = r;
  }
  const uint64_t L = off;
  res->total_bytes = L;
  for (int k = 0; k < 3; k++) res->tail_rank[k] = -1;
  const bool rs = (mode == SJB200_JSON_SEQUENCE_PARTIAL || mode == SJB200_JSON_SEQUENCE_FINAL);
  const bool is_final = (mode == SJB200_JSON_SEQUENCE_FINAL || mode == SJB200_COMMA_DELIMITED_FINAL);
  const bool unclosed = (final_state >> 1) & 1u;
  auto word = [&](int k, uint64_t p) {  // word p of the array after the in-place filter -> tail k
    if (p < W || p < T) {
      const bool f = p < W;
      int r = 0;
      while (!(f ? (p >= ranks[r].filtered_before && p < ranks[r].filtered_before + sums[r].filtered) : (p >= base[r] && p < base[r] + sums[r].count))) r++;
      res->tail_rank[k] = r;
      res->tail_pos[k] = uint32_t(p - (f ? ranks[r].filtered_before : base[r]));
      res->tail_filtered[k] = f ? 1u : 0u;
    } else {
      res->tail_val[k] = p < T + 2 ? uint32_t(L) : 0u;
    }
  };
  auto words_from = [&](uint64_t p) { for (int k = 0; k < 3; k++) word(k, p + uint64_t(k)); };
  auto done = [&](int err) {
    res->error = err;
    for (int r = 0; r < nranks && res->n_written; r++) {
      const uint64_t k = res->n > ranks[r].filtered_before ? res->n - ranks[r].filtered_before : 0;
      ranks[r].kept = std::min<uint64_t>(k, sums[r].filtered);
    }
    for (int r = 0, prev = -1; r < nranks; r++) {  // prev: the last earlier shard with kept entries
      if (ranks[r].kept == 0) continue;
      ranks[r].first_starts_document = (prev < 0) ? 1u : uint32_t(starts_document(sums[r].walk.role_first, sums[prev].walk.role_last));
      prev = r;
    }
    return err;
  };
  // find_next_document_index over the first k filtered entries
  auto walk = [&](uint64_t k) -> uint64_t {
    sjb200_stream_summary ws[kMaxRanks];
    for (int r = 0; r < nranks; r++) {
      const uint64_t fb = ranks[r].filtered_before;
      const uint64_t cnt = std::min<uint64_t>(k > fb ? k - fb : 0, sums[r].filtered);
      if (cnt == 0) memset(&ws[r], 0, sizeof(ws[r]));
      else ws[r] = (cnt == sums[r].filtered) ? sums[r].walk : sums[r].walk_below;
      ws[r].count = cnt;
      ws[r].len = sums[r].len;
    }
    sjb200_stream_fold_result fr;
    sjb200_stream_rank fk[kMaxRanks];
    sjb200_stream_fold(SJB200_STREAMING_FINAL, nranks, 0, 0, ws, &fr, fk);
    return fr.n;
  };
  if (flags_all & kFlagInternal) return done(SJB200_UNEXPECTED_ERROR);
  if (L == 0) return done(SJB200_UTF8_ERROR);                        // L198-204: nothing left after the trim
  if (flags_all & kFlagCtl) return done(SJB200_UNESCAPED_CHARS);    // L261-263
  res->n_written = 1;
  res->n = T;
  if (T == 0) { words_from(0); return done(SJB200_EMPTY); }          // L289-291
  if (!is_final && unclosed && T == 1) { res->n = 0; words_from(0); return done(SJB200_CAPACITY); }  // L298-302, before the filter
  uint64_t m = 0, n_res = W, next_start = L;
  bool too_large = false;
  const uint64_t last_sep = sep_rank >= 0 ? ranks[sep_rank].bytes_before + sums[sep_rank].last_sep : 0;
  const uint64_t before_sep = sep_rank >= 0 ? ranks[sep_rank].filtered_before + sums[sep_rank].below : 0;
  if (W != 0) {
    if (rs) {
      if (seps == 0) m = is_final ? walk(W) : 0;
      else if (is_final) m = W;
      else {
        next_start = last_sep;
        if (seps < 2) too_large = true;
        else m = before_sep;
      }
    } else {
      if (is_final) m = walk(W);
      else if (seps == 0) too_large = true;
      else {
        next_start = last_sep + 1;
        if (before_sep != 0) { n_res = before_sep; m = walk(before_sep); }
      }
    }
  }
  if (!is_final) {  // L344-359, L367-384
    if (too_large) { res->n = n_res; words_from(n_res); return done(SJB200_CAPACITY); }
    if (m == 0) { res->n = 0; words_from(0); return done(SJB200_EMPTY); }
    res->n = m;
    res->tail_val[0] = uint32_t(next_start);
    word(1, m + 1);
    word(2, m + 2);
  } else {  // L360-366, L385-393: word m + 1 = the old word m
    res->n = m;
    res->tail_val[0] = uint32_t(L);
    word(1, m);
    word(2, m + 2);
    if (m == 0) return done(SJB200_EMPTY);
  }
  return done((flags_all & kFlagUtf8) ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
}

extern "C" int sjb200_stage1_sharded_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx, void *stream) {
  return sharded_enqueue(m, kIndex, d_shard, len, last_shard, d_idx, nullptr, stream);
}

extern "C" int sjb200_stage1_sharded_finish(sjb200_comm *m, sjb200_sharded_result *out) { return sharded_finish(m, kIndex, out); }

extern "C" int sjb200_stage1_sharded(sjb200_comm *m, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx,
                                     sjb200_sharded_result *out, void *stream) {
  int rc = sjb200_stage1_sharded_enqueue(m, d_shard, len, last_shard, d_idx, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_stage1_sharded_finish(m, out);
}

extern "C" int sjb200_minify_sharded_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, uint8_t *d_dst, void *stream) {
  return sharded_enqueue(m, kMinify, d_shard, len, 0, nullptr, d_dst, stream);
}

extern "C" int sjb200_minify_sharded_finish(sjb200_comm *m, sjb200_sharded_result *out) { return sharded_finish(m, kMinify, out); }

extern "C" int sjb200_minify_sharded(sjb200_comm *m, const uint8_t *d_shard, size_t len, uint8_t *d_dst, sjb200_sharded_result *out, void *stream) {
  int rc = sjb200_minify_sharded_enqueue(m, d_shard, len, d_dst, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_minify_sharded_finish(m, out);
}

extern "C" int sjb200_validate_utf8_sharded_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, void *stream) {
  return sharded_enqueue(m, kUtf8, d_shard, len, 0, nullptr, nullptr, stream);
}

// returns 1 valid (every shard), 0 invalid, negative on a failure (CUDA, exchange timeout, kind mismatch)
extern "C" int sjb200_validate_utf8_sharded_finish(sjb200_comm *m, sjb200_sharded_result *out) {
  if (sharded_finish(m, kUtf8, out) != SJB200_SUCCESS) return -1;
  return (out->flags_all & kFlagUtf8) ? 0 : 1;
}

extern "C" int sjb200_validate_utf8_sharded(sjb200_comm *m, const uint8_t *d_shard, size_t len, sjb200_sharded_result *out, void *stream) {
  if (sjb200_validate_utf8_sharded_enqueue(m, d_shard, len, stream) != SJB200_SUCCESS) return -1;
  return sjb200_validate_utf8_sharded_finish(m, out);
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
