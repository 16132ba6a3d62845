// sjb200_capi.cu -- the C ABI (include/sjb200.h): contexts, options and stats, the single-GPU device-resident calls, the
// host-pointer pipeline, and the scan launches all of them and the sharded passes (sjb200_comm.cu) share.
// No torch, no CPU fallback: every scan runs in sjb200_kernels.cu or the call fails.
#include <ctype.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <new>

#include "sjb200_bits.cuh"
#include "sjb200_column.h"
#include "sjb200_column_double.h"
#include "sjb200_ctx.h"  // (with the CUDA runtime, include/sjb200.h and the launchers of sjb200_docs.cu and sjb200_tape.cu)
#include "sjb200_finish.h"
#include "sjb200_hostpipe.h"
#include "sjb200_kernels.cuh"
#include "sjb200_grammar.h"
#include "sjb200_pointer.h"

using namespace sjb200;

namespace {

size_t index_words(size_t capacity) { return ((capacity + 63) / 64) * 64 + 9; }
uint32_t tiles_of(size_t len) { return uint32_t((len + kTileBytes - 1) / kTileBytes); }

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
  const size_t n = std::max(need, size_t(tiles_of(c->capacity)) + 1);
  size_t words = 2 * c->desc_tiles;
  c->desc_tiles = 0;
  if (!grow(c, &c->d_count_desc, &words, 2 * n, "cudaMalloc(count_desc)")) return false;
  if (!ok(c, cudaMemsetAsync(c->d_count_desc, 0, 2 * n * sizeof(unsigned long long), c->stream), "memset desc")) return false;
  if (!ok(c, cudaStreamSynchronize(c->stream), "sync")) return false;
  c->desc_tiles = n;
  c->epoch = 0;
  return true;
}

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

// Enqueue the scan of document tiles [tile_begin, tile_begin+ntiles) of (d_buf,len).  carry_in null: the launch starts
// the document (zero state, zero count); has_last_tile: it scans the document's end.
bool enqueue_scan(sjb200_ctx *c, int kind, const CUtensorMap *map, bool tma, const uint8_t *d_buf, size_t len, uint32_t tile_begin,
                  uint32_t ntiles, bool has_last_tile, uint32_t *d_idx, uint8_t *d_dst, bool write_sentinels, const Carry *carry_in,
                  Carry *carry_out, Carry *carry_host, const Xchg *xchg, cudaStream_t stream, bool timed) {
  ScanParams p;
  memset(&p, 0, sizeof(p));
  p.buf = d_buf;
  p.len = len;
  p.pos_base = 0;
  p.prev_word = 0x20202020u;  // the document starts at byte 0 of d_buf
  p.check_eof = has_last_tile ? 1u : 0u;
  p.use_tma = tma ? 1u : 0u;
  p.tile_begin = tile_begin;
  p.ntiles = ntiles;
  if (!next_epoch(c, stream, &p.epoch)) return false;
  p.idx_out = d_idx;
  p.dst = d_dst;
  p.carry_in = carry_in;
  p.write_sentinels = write_sentinels ? 1u : 0u;
  p.carry_out = carry_out;
  p.carry_out_host = carry_host;
  p.flags = c->d_flags;
  p.count_desc = c->d_count_desc;
  p.ticket = c->d_ticket;
  if (xchg) p.xchg = *xchg;  // both kernels publish the record (scan4: stage 1 and minify; utf8v2: validate_utf8)
  p.debug = nullptr;
  if (c->opt_debug_timeline) {
    const uint32_t rows = std::max<uint32_t>(ntiles, 4096);  // (the trace build of scan4 writes 17 rows per CTA)
    grow(c, &c->d_debug, &c->debug_words, size_t(rows) * 8, "cudaMalloc(debug)");  // (without it the launch has no timeline)
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

}  // namespace

// ---- the scan helpers of sjb200_ctx.h
bool sjb200::ensure_desc(sjb200_ctx *c, size_t len) { return ensure_desc_n(c, tiles_of(len)); }

bool sjb200::scan_document(sjb200_ctx *c, int kind, const uint8_t *d_buf, size_t len, uint32_t *d_idx, uint8_t *d_dst, bool sentinels,
                           const Carry *carry_in, Carry *carry_out, Carry *carry_host, const Xchg *xchg, cudaStream_t stream, bool timed) {
  CUtensorMap map;
  bool tma = false;
  make_tensor_map(c, &map, d_buf, len, &tma);
  return enqueue_scan(c, kind, &map, tma, d_buf, len, 0, tiles_of(len), true, d_idx, d_dst, sentinels, carry_in, carry_out, carry_host, xchg, stream,
                      timed);
}

bool sjb200::fetch_result(sjb200_ctx *c, cudaStream_t s) {
  return ok(c, cudaMemcpyAsync(c->h_carry + 1, c->d_carry + 1, sizeof(Carry), cudaMemcpyDeviceToHost, s), "D2H result");
}

bool sjb200::trim_device_tail(sjb200_ctx *c, const uint8_t *d_buf, size_t *len, cudaStream_t s) {
  const size_t k = std::min<size_t>(3, *len);
  if (!ok(c, cudaMemcpyAsync(c->h_small, d_buf + *len - k, k, cudaMemcpyDeviceToHost, s), "D2H tail") || !ok(c, cudaStreamSynchronize(s), "sync"))
    return false;
  *len = trim_partial_utf8_tail(c->h_small, k, *len);
  return true;
}

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
  cudaFree(c->d_carry); cudaFree(c->d_flags); cudaFree(c->d_ticket); cudaFree(c->d_sfin); cudaFree(c->d_doc_scratch); cudaFree(c->d_ndocs); cudaFree(c->d_tok_scratch); cudaFree(c->d_tok_tot); cudaFree(c->d_tails); cudaFree(c->d_debug); cudaFree(c->d_doctab); cudaFree(c->d_stamps);
  cudaFree(c->d_ptr_blob); cudaFree(c->d_ptr_scratch); cudaFree(c->d_gram_scratch); cudaFree(c->d_col_scratch);
  if (c->h_ptr_blob) cudaFreeHost(c->h_ptr_blob);
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
    if (tail3) pc.len = trim_partial_utf8_tail(tail3, std::min<size_t>(3, len), len);
    else if (!trim_device_tail(c, d_buf, &pc.len, s)) { pc.early_error = SJB200_UNEXPECTED_ERROR; return false; }
    if (pc.len == 0) { pc.early_error = SJB200_UTF8_ERROR; return false; }
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
  // the kernel stores its result in the pinned host mirror itself
  if (!scan_document(c, kIndex, d_buf, len, d_idx, nullptr, true, nullptr, c->d_carry + slot, c->h_carry + slot, nullptr, s, true))
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
    if (!grow(c, &c->d_doc_scratch, &c->doc_scratch_words, filter_scratch_words(n), "cudaMalloc(filter scratch)")) return SJB200_MEMALLOC;
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
  stage1_enqueue_into(c, c->pending, d_buf, len, mode, d_idx, stream_of(c, stream), 1);
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
  if (off.back() > c->doctab_bytes) {  // the pinned half grows with the device half
    if (c->h_doctab) cudaFreeHost(c->h_doctab);
    c->h_doctab = nullptr;
    void *hp = nullptr;
    if (!grow(c, &c->d_doctab, &c->doctab_bytes, off.back(), "cudaMalloc(doc tables)") ||
        !ok(c, cudaMallocHost(&hp, off.back()), "cudaMallocHost(doc tables)")) {
      c->doctab_bytes = 0;
      return SJB200_MEMALLOC;
    }
    c->h_doctab = static_cast<uint8_t *>(hp);
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
    if (!grow(c, &c->d_stamps, &c->stamps_words, 2 * groups.size(), "cudaMalloc(stamps)")) return SJB200_MEMALLOC;
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
      if (!scan_document(c, kIndex, pc.d_buf, pc.len, pc.d_idx, nullptr, true, nullptr, c->d_carry + pc.carry_slot, c->h_carry + pc.carry_slot, nullptr, s,
                         false)) {
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
  cudaStream_t s = stream_of(c, stream);
  std::vector<PendingCall> calls;
  int done = 0;
  while (done < ndocs) {
    const int group = std::min(ndocs - done, kCarrySlots - 2);  // one result slot per document in flight
    calls.assign(size_t(group), PendingCall());
    const uint8_t *tails = nullptr;
    if (mode != SJB200_REGULAR) {
      // streaming modes look at every document's last three bytes before its scan (partial UTF-8 tail): fetch them for
      // the whole group with one launch and one copy instead of one synchronous copy per document
      const size_t need = size_t(group) * 20;
      if (c->tails_bytes < need) {  // the pinned half grows with the device half
        if (c->h_tails) cudaFreeHost(c->h_tails);
        c->h_tails = nullptr;
        void *hp = nullptr;
        if (!grow(c, &c->d_tails, &c->tails_bytes, need, "cudaMalloc(tails)") || !ok(c, cudaMallocHost(&hp, need), "cudaMallocHost(tails)")) {
          c->tails_bytes = 0;
          return SJB200_MEMALLOC;
        }
        c->h_tails = static_cast<uint8_t *>(hp);
      }
      const uint8_t **hptr = reinterpret_cast<const uint8_t **>(c->h_tails);
      uint64_t *hlen = reinterpret_cast<uint64_t *>(c->h_tails + size_t(group) * 8);
      uint8_t *hout = c->h_tails + size_t(group) * 16;
      for (int i = 0; i < group; i++) { hptr[i] = docs[done + i].d_buf; hlen[i] = (docs[done + i].len <= c->capacity) ? docs[done + i].len : 0; }
      const uint8_t *const *dptr = reinterpret_cast<const uint8_t *const *>(c->d_tails);
      const uint64_t *dlen = reinterpret_cast<const uint64_t *>(c->d_tails + size_t(group) * 8);
      uint8_t *dout = c->d_tails + size_t(group) * 16;
      if (!ok(c, cudaMemcpyAsync(c->d_tails, c->h_tails, size_t(group) * 16, cudaMemcpyHostToDevice, s), "H2D tail ptrs") ||
          !ok(c, launch_gather_tails(dptr, dlen, uint32_t(group), dout, s), "gather tails") ||
          !ok(c, cudaMemcpyAsync(hout, dout, size_t(group) * 4, cudaMemcpyDeviceToHost, s), "D2H tails") || !ok(c, cudaStreamSynchronize(s), "sync"))
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
  cudaStream_t s = stream_of(c, stream);
  if (!grow(c, &c->d_doc_scratch, &c->doc_scratch_words, doc_table_scratch_words(n), "cudaMalloc(doc scratch)")) return SJB200_MEMALLOC;
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
  cudaStream_t s = stream_of(c, stream);
  if (!grow(c, &c->d_tok_scratch, &c->tok_scratch_bytes, tokens_scratch_bytes(n), "cudaMalloc(token scratch)") ||
      (!c->d_tok_tot && !dev_alloc(c, &c->d_tok_tot, 1, "cudaMalloc(token totals)")))
    return SJB200_MEMALLOC;
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

// JSON Pointer lookup over the stage-2-lite tokens (dom::element::at_pointer for every document and pointer) --
// sjb200_pointer.cu
extern "C" int sjb200_at_pointer_dev(sjb200_ctx *c, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                     size_t string_bytes, const sjb200_doc_boundary *d_docs, uint32_t ndocs, const char *const *pointers,
                                     const size_t *pointer_lens, int npointers, sjb200_pointer_result *d_out, void *stream) {
  if (!c || npointers < 0 || (npointers && (!pointers || !pointer_lens || !d_out)) || (n && (!d_type || !d_payload)) ||
      (string_bytes && !d_strbuf))
    return SJB200_UNEXPECTED_ERROR;
  static_assert(sizeof(sjb200_pointer_result) == sizeof(ptr::PtrResult), "layout");
  ptr::CompiledPointers cp;
  const int rc = ptr::compile_pointers(pointers, pointer_lens, npointers, &cp);
  if (rc != SJB200_SUCCESS) return rc;
  if (npointers == 0) return SJB200_SUCCESS;
  if (!d_docs) ndocs = 0;
  DeviceGuard g(c->device);
  cudaStream_t s = stream_of(c, stream);
  // one blob [headers][levels][keys], copied in one transfer from pinned memory
  const size_t hb = cp.headers.size() * sizeof(ptr::PtrHeader), lb = cp.levels.size() * sizeof(ptr::PtrLevel);
  const size_t need = hb + lb + cp.keys.size() + 1;
  if (c->ptr_blob_bytes < need) {
    if (c->h_ptr_blob) cudaFreeHost(c->h_ptr_blob);
    c->h_ptr_blob = nullptr;
    c->ptr_blob_bytes = 0;
    cudaFree(c->d_ptr_blob);
    c->d_ptr_blob = nullptr;
    if (!ok(c, cudaMallocHost(&c->h_ptr_blob, need), "cudaMallocHost(pointers)") || !dev_alloc(c, &c->d_ptr_blob, need, "cudaMalloc(pointers)"))
      return SJB200_MEMALLOC;
    c->ptr_blob_bytes = need;
  }
  memcpy(c->h_ptr_blob, cp.headers.data(), hb);
  memcpy(c->h_ptr_blob + hb, cp.levels.data(), lb);
  memcpy(c->h_ptr_blob + hb + lb, cp.keys.data(), cp.keys.size());
  if (!grow(c, &c->d_ptr_scratch, &c->ptr_scratch_words, ptr::pointer_scratch_words(ndocs ? ndocs : 1), "cudaMalloc(pointer scratch)"))
    return SJB200_MEMALLOC;
  ptr::PtrLaunch a{};
  a.w = ptr::Walk{d_type, d_payload, d_strbuf, string_bytes, reinterpret_cast<const ptr::PtrLevel *>(c->d_ptr_blob + hb), c->d_ptr_blob + hb + lb};
  a.n = n;
  a.docs = ndocs ? reinterpret_cast<const sjb200_doc_boundary_t *>(d_docs) : nullptr;
  a.ndocs = ndocs;
  a.headers = reinterpret_cast<const ptr::PtrHeader *>(c->d_ptr_blob);
  a.npointers = uint32_t(npointers);
  a.out = reinterpret_cast<ptr::PtrResult *>(d_out);
  if (!ok(c, cudaMemcpyAsync(c->d_ptr_blob, c->h_ptr_blob, need, cudaMemcpyHostToDevice, s), "H2D pointers") ||
      !ok(c, ptr::launch_at_pointer(a, c->d_ptr_scratch, c->sm_count, s), "at_pointer") || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += 3;
  return SJB200_SUCCESS;
}

// Typed columns from JSON Pointer results (element::get_int64 / get_uint64 / get_bool / get_string and container sizes
// of every row) -- sjb200_column.cu
extern "C" int sjb200_column_dev(sjb200_ctx *c, int kind, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                 size_t string_bytes, const sjb200_pointer_result *d_rows, uint32_t nrows, int32_t *d_err, uint8_t *d_row_type,
                                 void *d_values, int64_t *d_offsets, uint8_t *d_bytes, size_t bytes_capacity, sjb200_column_result *out, void *stream) {
  if (!c || !out || kind < SJB200_COLUMN_INT64 || kind > SJB200_COLUMN_OBJECT_SIZE) return SJB200_UNEXPECTED_ERROR;
  out->rows_in_error = 0;
  out->reserved = 0;
  out->string_bytes = 0;
  const bool str = kind == SJB200_COLUMN_STRING;
  if ((n && (!d_type || !d_payload)) || (string_bytes && !d_strbuf) || (str && !d_offsets) ||
      (nrows && (!d_rows || !d_err || !d_row_type || (!str && !d_values))) || (str && bytes_capacity && !d_bytes))
    return SJB200_UNEXPECTED_ERROR;
  static_assert(sizeof(sjb200_pointer_result) == sizeof(col::Row), "layout");
  DeviceGuard g(c->device);
  cudaStream_t s = stream_of(c, stream);
  if (!grow(c, &c->d_col_scratch, &c->col_scratch_words, (col::column_scratch_bytes(nrows, str ? bytes_capacity : 0) + 7) / 8, "cudaMalloc(column scratch)")) return SJB200_MEMALLOC;
  col::ColLaunch a{};
  a.c = col::Cols{d_type, d_payload, n, d_strbuf, string_bytes, reinterpret_cast<const col::Row *>(d_rows), nrows};
  a.kind = kind;
  a.err = d_err;
  a.row_type = d_row_type;
  a.values = d_values;
  a.offsets = d_offsets;
  a.bytes = d_bytes;
  a.bytes_capacity = str ? bytes_capacity : 0;
  TokenTotals *tot = nullptr;
  int launches = 0;
  if (!ok(c, col::launch_column(a, c->d_col_scratch, &tot, c->sm_count, s, &launches), "column") ||
      !ok(c, cudaMemcpyAsync(c->h_small, tot, sizeof(TokenTotals), cudaMemcpyDeviceToHost, s), "D2H column totals") || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += launches;
  TokenTotals t;
  memcpy(&t, c->h_small, sizeof(t));
  out->rows_in_error = t.n_strings;
  if (str) out->string_bytes = t.string_bytes;
  return str && t.string_bytes > bytes_capacity ? SJB200_CAPACITY : SJB200_SUCCESS;
}

// element::get_double of every row of JSON Pointer results -- sjb200_column_double.cu
extern "C" int sjb200_column_double_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, const uint32_t *d_idx, const uint8_t *d_type,
                                        const uint64_t *d_payload, uint32_t n, const sjb200_pointer_result *d_rows, uint32_t nrows, int32_t *d_err,
                                        uint8_t *d_row_type, double *d_values, sjb200_column_result *out, void *stream) {
  if (!c || !out) return SJB200_UNEXPECTED_ERROR;
  out->rows_in_error = 0;
  out->reserved = 0;
  out->string_bytes = 0;
  if ((n && (!d_type || !d_payload || !d_idx)) || (len && !d_buf) || (nrows && (!d_rows || !d_err || !d_row_type || !d_values))) return SJB200_UNEXPECTED_ERROR;
  if (nrows == 0) return SJB200_SUCCESS;
  static_assert(sizeof(sjb200_pointer_result) == sizeof(col::Row), "layout");
  DeviceGuard g(c->device);
  cudaStream_t s = stream_of(c, stream);
  if (!grow(c, &c->d_col_scratch, &c->col_scratch_words, (dbl::column_double_scratch_bytes(nrows) + 7) / 8, "cudaMalloc(column scratch)")) return SJB200_MEMALLOC;
  dbl::DoubleLaunch a{};
  a.c = col::Cols{d_type, d_payload, n, nullptr, 0, reinterpret_cast<const col::Row *>(d_rows), nrows};
  a.buf = d_buf;
  a.len = len;
  a.idx = d_idx;
  a.err = d_err;
  a.row_type = d_row_type;
  a.values = reinterpret_cast<uint64_t *>(d_values);
  uint32_t *counts = nullptr;
  int launches = 0;
  if (!ok(c, dbl::launch_column_double(a, c->d_col_scratch, &counts, c->sm_count, s, &launches), "column double") ||
      !ok(c, cudaMemcpyAsync(c->h_small, counts, sizeof(uint32_t), cudaMemcpyDeviceToHost, s), "D2H column double totals") || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += launches;
  uint32_t rows_in_error;
  memcpy(&rows_in_error, c->h_small, sizeof(rows_in_error));
  out->rows_in_error = rows_in_error;
  return SJB200_SUCCESS;
}

// Stage-2 grammar over the stage-2-lite tokens (the error walk_document returns for every document) -- sjb200_grammar.cu
extern "C" int sjb200_document_errors_dev(sjb200_ctx *c, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const sjb200_doc_boundary *d_docs,
                                          uint32_t ndocs, size_t max_depth, sjb200_document_error *d_out, sjb200_document_errors_result *out,
                                          void *stream) {
  if (!c || !d_out || !out || (n && (!d_type || !d_payload))) return SJB200_UNEXPECTED_ERROR;
  if (max_depth == 0 || max_depth > SJB200_DOCUMENT_MAX_DEPTH) return SJB200_CAPACITY;
  static_assert(sizeof(sjb200_document_error) == sizeof(gram::DocError), "layout");
  static_assert(SJB200_DOCUMENT_MAX_DEPTH == gram::kMaxDepth, "limit");
  if (!d_docs) ndocs = 0;
  DeviceGuard g(c->device);
  cudaStream_t s = stream_of(c, stream);
  const size_t words = gram::grammar_scratch_words(n, ndocs, uint32_t(max_depth));
  if (!grow(c, &c->d_gram_scratch, &c->gram_scratch_words, words + 4, "cudaMalloc(grammar scratch)")) return SJB200_MEMALLOC;
  gram::GrammarArgs a{};
  a.type = d_type;
  a.payload = d_payload;
  a.n = n;
  a.docs = ndocs ? reinterpret_cast<const sjb200_doc_boundary_t *>(d_docs) : nullptr;
  a.ndocs = ndocs;
  a.max_depth = uint32_t(max_depth);
  a.out = reinterpret_cast<gram::DocError *>(d_out);
  uint32_t *summary = c->d_gram_scratch + words;
  int launched = 0;
  if (!ok(c, gram::launch_document_errors(a, c->d_gram_scratch, summary, c->sm_count, s, &launched), "document_errors") ||
      !ok(c, cudaMemcpyAsync(c->h_small, summary, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s), "D2H summary") ||
      !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += unsigned(launched);
  uint32_t sum[3];
  memcpy(sum, c->h_small, sizeof(sum));
  out->ndocs_in_error = sum[1];
  out->first_doc_in_error = sum[2];
  return sum[0] ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
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
  cudaStream_t s = stream_of(c, stream);
  PendingCall &pc = c->pending;
  pc = PendingCall();
  pc.kind = kMinify; pc.d_buf = d_buf; pc.d_dst = d_dst; pc.stream = s; pc.len = len;
  if (len > kMaxBytes) { pc.early_error = SJB200_CAPACITY; return SJB200_SUCCESS; }
  if (len == 0) { pc.early_error = SJB200_SUCCESS; return SJB200_SUCCESS; }  // json_minifier.h: nothing to do, dst_len = 0
  if (!ensure_desc(c, len)) { pc.early_error = SJB200_MEMALLOC; return SJB200_SUCCESS; }
  if (!scan_document(c, kMinify, d_buf, len, nullptr, d_dst, false, nullptr, c->d_carry + 1, nullptr, nullptr, s, true) ||
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
  cudaStream_t s = stream_of(c, stream);
  PendingCall &pc = c->pending;
  pc = PendingCall();
  pc.kind = kUtf8; pc.d_buf = d_buf; pc.stream = s; pc.len = len;
  if (len == 0) { pc.early_error = SJB200_SUCCESS; return SJB200_SUCCESS; }  // utf8_validator.h L27-28: empty is valid
  if (len > kMaxBytes) { pc.early_error = SJB200_CAPACITY; return SJB200_SUCCESS; }
  if (!scan_document(c, kUtf8, d_buf, len, nullptr, nullptr, false, nullptr, c->d_carry + 1, nullptr, nullptr, s, true) ||
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
bool ensure_input(sjb200_ctx *c, size_t len) { return grow(c, &c->d_in, &c->d_in_bytes, std::max(len, c->capacity) + 256, "cudaMalloc(input)"); }
bool ensure_index(sjb200_ctx *c, size_t len) { return grow(c, &c->d_idx, &c->d_idx_words, index_words(std::max(len, c->capacity)), "cudaMalloc(index)"); }
bool ensure_output(sjb200_ctx *c, size_t len) { return grow(c, &c->d_out, &c->d_out_bytes, len + 256, "cudaMalloc(output)"); }

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
    if (!enqueue_scan(c, kind, &map, tma, c->d_in, len, uint32_t(off / kTileBytes), tiles_of(bytes), last, d_idx, d_dst, false,
                      k == 0 ? nullptr : c->d_carry + k, c->d_carry + k + 1, c->h_carry + k + 1, nullptr, c->stream, true))
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
