// sjb200_comm.cu -- shards of one document or stream across GPUs: the per-shard scans (sjb200_stage1_shard_dev*) and the
// sharded passes of every kind on a sjb200_comm, with the exchange fused into their kernels.  Their host folds are in
// sjb200_fold.cpp.
#include <string.h>

#include <chrono>
#include <new>

#include "sjb200_bits.cuh"
#include "sjb200_ctx.h"
#include "sjb200_grammar.h"
#include "sjb200_kernels.cuh"
#include "sjb200_pointer.h"

using namespace sjb200;

namespace {

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// stream and delimited passes scan like stage 1; only their records' kind differs
int scan_kind_of(int kind) { return (kind == kStream || kind == kDelim) ? kIndex : kind; }

// Scan the whole shard again from a known incoming state: carry slot 0 holds that state and count 0, so the output starts
// at d_idx[0] / d_dst[0].  The result comes back in h_carry[1].
int scan_from_state(sjb200_ctx *c, int kind, const uint8_t *d_buf, size_t len, uint32_t state_in, uint32_t *d_idx, uint8_t *d_dst, cudaStream_t s) {
  if (!ensure_desc(c, len)) return SJB200_MEMALLOC;
  c->h_carry[0] = Carry{0, state_in & 7u, 0, 0, 0};
  if (!ok(c, cudaMemcpyAsync(c->d_carry, c->h_carry, sizeof(Carry), cudaMemcpyHostToDevice, s), "H2D carry") ||
      !scan_document(c, kind, d_buf, len, d_idx, d_dst, false, c->d_carry, c->d_carry + 1, nullptr, nullptr, s, true) ||
      !fetch_result(c, s) || !ok(c, cudaStreamSynchronize(s), "sync"))
    return SJB200_UNEXPECTED_ERROR;
  return SJB200_SUCCESS;
}

}  // namespace

extern "C" int sjb200_stage1_shard_dev(sjb200_ctx *c, const uint8_t *d_buf, size_t len, uint32_t state_in, int last_shard,
                                       uint32_t *d_idx, sjb200_shard_result *out, void *stream) {
  if (!c || !out) return SJB200_UNEXPECTED_ERROR;
  memset(out, 0, sizeof(*out));
  if (len == 0 || len > kMaxBytes) return SJB200_UNEXPECTED_ERROR;
  DeviceGuard g(c->device);
  (void)last_shard;  // every shard checks its own end: cuts are at character boundaries (sjb200_shard_cut)
  const int rc = scan_from_state(c, kIndex, d_buf, len, state_in, d_idx, nullptr, stream_of(c, stream));
  if (rc != SJB200_SUCCESS) return rc;
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
  if (!ensure_desc(c, len)) return SJB200_MEMALLOC;
  if (!scan_document(c, kIndex, d_buf, len, d_idx, nullptr, false, nullptr, static_cast<Carry *>(d_result), nullptr, nullptr, stream_of(c, stream), true))
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
  unsigned long long *h_rec = nullptr;             // pinned [kMaxRanks][kGramWords]: records ([r][0..1]), summaries, delimited or grammar blocks
  uint32_t *h_tot = nullptr;                       // pinned [4]: a delimited pass's filter totals
  uint32_t *d_scratch = nullptr;                   // a delimited pass's filter scratch (delim_scratch_words)
  size_t scratch_words = 0;
  Carry *d_result = nullptr;                       // [kXchgSteps] the launches' own result blocks
  // tokens passes, by the slot of their pass (a pass in flight keeps its own): totals, tile scratch (grow-only)
  TokenTotals *d_tok_tot = nullptr;
  uint8_t *d_tok_scratch[kXchgSteps] = {};
  size_t tok_scratch_bytes[kXchgSteps] = {};
  // grammar passes, by the slot of their pass: the call's arguments, scratch (grow-only)
  struct GramStep {
    const uint8_t *type; const uint64_t *payload; uint32_t n; bool whole; const sjb200_doc_boundary *docs; uint32_t ndocs; size_t max_depth;
    sjb200_sharded_document_error *out;
  } gram[kXchgSteps];
  uint32_t *d_gram_scratch[kXchgSteps] = {};
  size_t gram_scratch_words[kXchgSteps] = {};
  // pointer passes, by the slot of their pass: the launch (with the compiled pointers' device copy), scratch (grow-only)
  struct PtrStep {
    ptr::PtrShard s;
    bool whole;
  } ptrs[kXchgSteps];
  uint8_t *d_ptr_blob[kXchgSteps] = {};
  size_t ptr_blob_bytes[kXchgSteps] = {};
  uint32_t *d_ptr_scratch[kXchgSteps] = {};
  size_t ptr_scratch_words[kXchgSteps] = {};
  cudaStream_t poll_stream = nullptr;
  cudaEvent_t done[kXchgSteps] = {};
  struct Step {
    const uint8_t *d_buf; size_t len; uint32_t *d_idx; uint8_t *d_dst; cudaStream_t stream; uint32_t seq; int last; int kind; int mode;
    std::chrono::steady_clock::time_point t_enq;  // when its enqueue began (stat xchg_enqueue_ms)
  } steps[kXchgSteps];
  uint32_t head = 0, tail = 0;                     // passes enqueued / finished
  long poll_timeout_ms = 20000;
};

namespace {
constexpr size_t kWindowWords = kXchgWindowWords;
constexpr size_t kHostWords = size_t(kMaxRanks) * (kGramWords > kDelimWords ? kGramWords : kDelimWords);  // h_rec
uint32_t window_slot(uint32_t seq, int round) { return (seq % uint32_t(kXchgSteps)) * 2u + uint32_t(round); }

// Where this rank's launches of pass `seq` store their words.  Rounds 0 and 1 are records, in their window slot; the
// summary (2) and delimited (3) rounds' kernels store at a word offset of their own.
Xchg comm_target(const sjb200_comm *m, uint32_t seq, int round) {
  Xchg x;
  memset(&x, 0, sizeof(x));
  for (int r = 0; r < kMaxRanks; r++) x.peer[r] = m->peer[r];
  x.nranks = uint32_t(m->nranks); x.rank = uint32_t(m->rank); x.seq = seq;
  if (round < 2) x.slot = window_slot(seq, round);
  return x;
}

// wait (host polling, bounded) until every rank's record of (seq, round) is in the local window; records -> comm->h_rec.
// round 2: the summaries of a streaming pass (kSumWords words per rank, each tagged with seq).  round 3: words
// [first, first + nwords) of every rank's delimited block (h_rec[r * kDelimWords + k], the whole blocks are copied).
// round 4: the same of every rank's grammar block (h_rec[r * kGramWords + k]).
int comm_collect(sjb200_comm *m, uint32_t seq, int round, int first = 0, int nwords = 0) {
  sjb200_ctx *c = m->ctx;
  const bool sums = (round == 2), gram = (round == 4), delim = (round == 3) || gram;
  const unsigned long long *src = gram   ? m->window + xchg_gram_at(seq, 0)
                                  : delim ? m->window + xchg_delim_at(seq, 0)
                                  : sums ? m->window + xchg_summary_at(seq, 0)
                                         : m->window + size_t(window_slot(seq, round)) * kMaxRanks * 2;
  const size_t words = gram ? size_t(kGramWords) : delim ? size_t(kDelimWords) : sums ? size_t(kSumWords) : 2;
  const auto t0 = std::chrono::steady_clock::now();
  for (;;) {
    if (!ok(c, cudaMemcpyAsync(m->h_rec, src, size_t(m->nranks) * words * 8, cudaMemcpyDeviceToHost, m->poll_stream), "D2H window") ||
        !ok(c, cudaStreamSynchronize(m->poll_stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->xchg_polls++;
    bool all = true;
    for (int r = 0; r < m->nranks; r++) {
      if (delim) {
        for (int k = first; k < first + nwords; k++) all = all && uint32_t(m->h_rec[size_t(r) * words + k] >> 32) == seq;
        continue;
      }
      if (!sums) { all = all && xchg_complete(m->h_rec[2 * r], m->h_rec[2 * r + 1], seq); continue; }
      for (int k = 0; k < kSumWords; k++) all = all && uint32_t(m->h_rec[size_t(r) * kSumWords + k] >> 32) == seq;
    }
    if (all) {
      c->xchg_wait_ms += ms_since(t0);
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
              ok(c, cudaMallocHost(&hp, kHostWords * 8 + 16), "cudaMallocHost") &&
              ok(c, cudaStreamCreateWithFlags(&m->poll_stream, cudaStreamNonBlocking), "stream");
  m->h_rec = static_cast<unsigned long long *>(hp);
  if (hp) m->h_tot = reinterpret_cast<uint32_t *>(m->h_rec + kHostWords);
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
  for (uint8_t *p : m->d_tok_scratch) cudaFree(p);
  for (uint32_t *p : m->d_gram_scratch) cudaFree(p);
  for (uint8_t *p : m->d_ptr_blob) cudaFree(p);
  for (uint32_t *p : m->d_ptr_scratch) cudaFree(p);
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
// The first half of every sharded enqueue: the pass's Step, or null when kXchgSteps / 2 passes are in flight already
// (CAPACITY: finish some first).  Its seq is head + 1: tags start at 1, so a zeroed window never matches.
sjb200_comm::Step *pass_begin(sjb200_comm *m, int kind, int mode, int last, const uint8_t *d_buf, size_t len, uint32_t *d_idx, uint8_t *d_dst,
                              void *stream) {
  if (m->head - m->tail >= uint32_t(kXchgSteps / 2)) return nullptr;
  sjb200_comm::Step &st = m->steps[m->head % uint32_t(kXchgSteps)];
  st = sjb200_comm::Step{d_buf, len, d_idx, d_dst, stream_of(m->ctx, stream), m->head + 1, last, kind, mode, std::chrono::steady_clock::now()};
  return &st;
}

// The second half: the event that marks the end of the pass's launches on its stream; the pass is then in flight.
int pass_end(sjb200_comm *m, bool launched) {
  sjb200_ctx *c = m->ctx;
  const uint32_t i = m->head % uint32_t(kXchgSteps);
  if (!launched || !ok(c, cudaEventRecord(m->done[i], m->steps[i].stream), "event record")) return SJB200_UNEXPECTED_ERROR;
  m->head++;
  c->xchg_enqueue_ms += ms_since(m->steps[i].t_enq);
  return SJB200_SUCCESS;
}

// The first half of every sharded finish (the caller has checked that a pass is in flight): the oldest pass must be of
// `kind` -- else it stays in flight, and the caller can still finish it with the right call.  Then its launches are
// waited for, and round 0 brings every rank's record, which must be of `kind` too.  *st: the pass.
int pass_pop(sjb200_comm *m, int kind, sjb200_comm::Step *st) {
  sjb200_ctx *c = m->ctx;
  const uint32_t i = m->tail % uint32_t(kXchgSteps);
  if (m->steps[i].kind != kind) {
    c->last_error = "sharded finish: the oldest pass in flight is of another kind";
    return SJB200_UNEXPECTED_ERROR;
  }
  *st = m->steps[i];
  m->tail++;
  const auto t_ev = std::chrono::steady_clock::now();
  if (!ok(c, cudaEventSynchronize(m->done[i]), "event sync")) return SJB200_UNEXPECTED_ERROR;  // own launches (and their stores) done
  c->xchg_evsync_ms += ms_since(t_ev);
  const int rc = comm_collect(m, st->seq, 0);
  if (rc != SJB200_SUCCESS) return rc;
  for (int r = 0; r < m->nranks; r++)
    if (xchg_kind(m->h_rec[2 * r + 1]) != kind) {  // never fold one kind's counts into another's base
      c->last_error = "sharded pass " + std::to_string(st->seq) + ": rank " + std::to_string(r) + " published a pass of another kind (every rank must enqueue the same sequence of kinds)";
      return SJB200_UNEXPECTED_ERROR;
    }
  return SJB200_SUCCESS;
}

// Enqueue one pass of `kind` (kIndex, kStream, kDelim: d_idx, kMinify: d_dst, kUtf8: neither).  The launch's record lands in
// every rank's window.
int sharded_enqueue(sjb200_comm *m, int kind, const uint8_t *d_shard, size_t len, int last_shard, uint32_t *d_idx, uint8_t *d_dst, void *stream,
                    int mode = SJB200_REGULAR) {
  const int scan_kind = scan_kind_of(kind);
  if (!m || !m->connected || !d_shard || len == 0 || len > kMaxBytes || (scan_kind == kIndex && !d_idx) || (kind == kMinify && !d_dst))
    return SJB200_UNEXPECTED_ERROR;
  if (kind == kStream && (mode < SJB200_REGULAR || mode > SJB200_STREAMING_FINAL)) return SJB200_UNEXPECTED_ERROR;
  if (kind == kDelim && (mode < SJB200_JSON_SEQUENCE_PARTIAL || mode > SJB200_COMMA_DELIMITED_FINAL)) return SJB200_UNEXPECTED_ERROR;
  sjb200_comm::Step *st = pass_begin(m, kind, mode, last_shard, d_shard, len, d_idx, d_dst, stream);
  if (!st) return SJB200_CAPACITY;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  if ((kind == kStream || kind == kDelim) && last_shard && mode != SJB200_REGULAR && !trim_device_tail(c, d_shard, &st->len, st->stream))
    return SJB200_UNEXPECTED_ERROR;  // (the stream's end)
  if (scan_kind != kUtf8 && st->len && !ensure_desc(c, st->len)) return SJB200_MEMALLOC;  // (scan4's look-back descriptors)
  Xchg x = comm_target(m, st->seq, 0);
  x.kind = uint32_t(kind);
  bool good;
  if (st->len == 0) {  // a last shard that trims to nothing: no scan; its record {count 0, escape passed through, no flags}
    good = ok(c, launch_xchg_post(x, xchg_word0(st->seq, 0), xchg_word1(st->seq, 0, 0x8u, 0, kind), st->stream), "xchg post");
    c->launches += good ? 1 : 0;
  } else {
    good = scan_document(c, scan_kind, d_shard, st->len, d_idx, d_dst, false, nullptr, m->d_result + m->head % uint32_t(kXchgSteps), nullptr, &x,
                         st->stream, true);
  }
  return pass_end(m, good);
}

// Complete the oldest pass in flight, which must be of `kind`: the one body of the three sharded finishes.  *pass: the pass.
int sharded_finish(sjb200_comm *m, int kind, sjb200_sharded_result *out, sjb200_comm::Step *pass = nullptr) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  memset(out, 0, sizeof(*out));
  sjb200_comm::Step st;
  int rc = pass_pop(m, kind, &st);
  if (rc != SJB200_SUCCESS) return rc;
  if (pass) *pass = st;
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
      rc = scan_from_state(c, scan_kind_of(kind), st.d_buf, st.len, my_state, st.d_idx, st.d_dst, st.stream);
      if (rc != SJB200_SUCCESS) return rc;
      my_count = c->h_carry[1].count;
      // (as in the kernel's record: an internal error is the only flag that means something to minify)
      my_flags = c->h_carry[1].flags & (kind == kMinify ? uint32_t(kFlagInternal) : ~0u);
      if (my_flags & kFlagInternal) return SJB200_UNEXPECTED_ERROR;
      out->rescanned = 1;
    }
    if (!ok(c, launch_xchg_post(comm_target(m, st.seq, 1), xchg_word0(st.seq, my_count), xchg_word1(st.seq, out->state_out, tt[m->rank], my_flags, kind),
                                st.stream), "xchg post") ||
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

// every rank's count from the records in h_rec (the second round's, if it ran); returns the rank that holds the stream's
// last structural (-1: none)
int holder_and_counts(const sjb200_comm *m, uint64_t *counts) {
  int holder = -1;
  for (int r = 0; r < m->nranks; r++) {
    counts[r] = xchg_count(m->h_rec[2 * r]);
    if (counts[r]) holder = r;
  }
  return holder;
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
  sjb200_comm::Step st;
  int rc = sharded_finish(m, kStream, &out->shard, &st);
  if (rc != SJB200_SUCCESS) return rc;  // (an internal error is seen by every rank alike: nobody runs the summary round)
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  uint64_t counts[kMaxRanks];
  const int holder = holder_and_counts(m, counts);
  const bool unclosed = (out->shard.final_state >> 1) & 1u;
  const uint64_t my_count = counts[m->rank];
  const uint64_t kept = my_count - ((st.mode != SJB200_REGULAR && unclosed && holder == m->rank) ? 1 : 0);
  if (!ok(c, launch_stream_summary(st.d_buf, st.d_idx, uint32_t(my_count), uint32_t(kept), uint32_t(st.len), st.mode != SJB200_REGULAR,
                                   comm_target(m, st.seq, 2), xchg_summary_at(st.seq, uint32_t(m->rank)), m->poll_stream),
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

// Complete the oldest pass in flight, a delimited pass (modes 3..6): the scan's fold (sharded_finish), then three rounds,
// each a small kernel storing tagged words into every rank's window and a comm_collect (DESIGN.md section 5):
//   carry   every rank's length and the bracket net (comma) or "ends inside a separator run" / "whitespace / RS only"
//           (RS) -> this rank's depth_in / run_in;
//   filter  the filter of sjb200_docs.cu with that carry, into the scratch, then its totals and the walks of
//           find_next_document_index over the filtered entries -> sjb200_delimited_fold;
//   tail    the holders of the words n, n+1, n+2 publish them (skipped when the fold knows all three); then the
//           filtered entries go back into d_idx.
int sharded_delimited_finish(sjb200_comm *m, sjb200_sharded_delimited_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  memset(out, 0, sizeof(*out));
  sjb200_comm::Step st;
  int rc = sharded_finish(m, kDelim, &out->stream.shard, &st);
  if (rc != SJB200_SUCCESS) return rc;  // (an internal error is seen by every rank alike: nobody runs the extra rounds)
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const int me = m->rank;
  uint64_t counts[kMaxRanks];
  const int holder = holder_and_counts(m, counts);
  const bool unclosed = (out->stream.shard.final_state >> 1) & 1u;
  const bool comma = (st.mode == SJB200_COMMA_DELIMITED_PARTIAL || st.mode == SJB200_COMMA_DELIMITED_FINAL);
  const bool walk_below = (st.mode == SJB200_COMMA_DELIMITED_PARTIAL);
  // the structurals this shard's filter considers: less the stream's last one when it ends inside a string
  const uint32_t n = uint32_t(counts[me]) - ((unclosed && holder == me) ? 1u : 0u);
  const uint32_t len = uint32_t(st.len);
  if (!grow(c, &m->d_scratch, &m->scratch_words, delim_scratch_words(n), "cudaMalloc(delimited scratch)")) return SJB200_MEMALLOC;
  const Xchg x = comm_target(m, st.seq, 3);
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

// ---------------------------------------------------------------------------------------------- sharded stage-2-lite
// Enqueue one tokens pass: the launches of sjb200_tokens_dev on the shard, on the totals and tile scratch of the pass's
// own slot (passes of every kind may be in flight), with tile_scan_kernel storing the record and the summary into every
// rank's window.  A rank that cannot run its pass (device allocation) still publishes a record, with kFlagInternal, so
// that every rank's finish fails alike instead of waiting for it.
extern "C" int sjb200_tokens_sharded_enqueue(sjb200_comm *m, const uint8_t *d_shard, size_t len, uint32_t state_in, const uint32_t *d_idx, uint32_t n,
                                             uint8_t *d_type, uint64_t *d_payload, uint8_t *d_strbuf, size_t strbuf_capacity, void *stream) {
  if (!m || !m->connected || len > kMaxBytes || state_in > 7u || (n && (!d_shard || !d_idx || !d_type || !d_payload)) || (strbuf_capacity && !d_strbuf))
    return SJB200_UNEXPECTED_ERROR;
  sjb200_comm::Step *st = pass_begin(m, kTokens, 0, 0, d_shard, len, nullptr, nullptr, stream);
  if (!st) return SJB200_CAPACITY;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const uint32_t i = m->head % uint32_t(kXchgSteps);
  const TokXchg x{comm_target(m, st->seq, 0), state_in, n, len, strbuf_capacity};
  // (the slot's previous pass has been finished: at most kXchgSteps / 2 are in flight)
  const bool have = (m->d_tok_tot || dev_alloc(c, &m->d_tok_tot, kXchgSteps, "cudaMalloc(token totals)")) &&
                    grow(c, &m->d_tok_scratch[i], &m->tok_scratch_bytes[i], tokens_scratch_bytes(n), "cudaMalloc(token scratch)");
  bool good;
  if (have) {
    good = ok(c, launch_tokens(d_shard, len, d_idx, n, d_type, d_payload, d_strbuf, strbuf_capacity, m->d_tok_scratch[i], m->d_tok_tot + i,
                               int(c->opt_tok_stage), st->stream, &x), "tokens");
    c->launches += good ? (n ? 3 : 1) : 0;
  } else {
    good = ok(c, launch_xchg_post(x.xchg, xchg_word0(st->seq, 0), xchg_word1(st->seq, state_in, 0, kFlagInternal, kTokens), st->stream), "xchg post");
    c->launches += good ? 1 : 0;
  }
  return pass_end(m, good);
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
  sjb200_comm::Step st;
  int rc = pass_pop(m, kTokens, &st);
  if (rc != SJB200_SUCCESS) return rc;
  int failed = -1;
  for (int r = 0; r < m->nranks; r++) {
    const unsigned long long w1 = m->h_rec[2 * r + 1];
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

// ---------------------------------------------------------------------------------------------- sharded stage-2 grammar
// Enqueue one grammar pass: the table's check and start bitmap, then the edge words and the round-0 record into every
// rank's window.  Passes A-C wait for finish, which knows the halo.  A rank that cannot run its pass (bad arguments,
// device allocation) still publishes, flagged, so that every rank's finish fails alike instead of waiting for it.
extern "C" int sjb200_document_errors_sharded_enqueue(sjb200_comm *m, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, int whole,
                                                      const sjb200_doc_boundary *d_docs, uint32_t ndocs, size_t max_depth,
                                                      sjb200_sharded_document_error *d_out, void *stream) {
  if (!m || !m->connected) return SJB200_UNEXPECTED_ERROR;
  sjb200_comm::Step *st = pass_begin(m, kGrammar, 0, 0, nullptr, 0, nullptr, nullptr, stream);
  if (!st) return SJB200_CAPACITY;
  static_assert(sizeof(sjb200_sharded_document_error) == sizeof(gram::sjb200_sharded_document_error_t), "layout");
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const uint32_t i = m->head % uint32_t(kXchgSteps);
  if (whole) ndocs = 0;
  bool failed = (n && (!d_type || !d_payload)) || (ndocs && !d_docs) || (!d_out && (whole ? m->rank == 0 : ndocs > 0));
  if (failed) c->last_error = "sharded grammar pass: bad arguments";
  const uint32_t md = max_depth == 0 ? 1u : max_depth > gram::kMaxDepth ? gram::kMaxDepth : uint32_t(max_depth);  // (CAPACITY is decided in finish)
  gram::GrammarArgs a{};
  a.type = d_type; a.payload = d_payload; a.n = n;
  a.docs = ndocs ? reinterpret_cast<const sjb200_doc_boundary_t *>(d_docs) : nullptr;
  a.ndocs = ndocs; a.max_depth = md;
  failed = failed || !grow(c, &m->d_gram_scratch[i], &m->gram_scratch_words[i], gram::shard_scratch_words(n, ndocs, md), "cudaMalloc(grammar scratch)");
  m->gram[i] = sjb200_comm::GramStep{d_type, d_payload, n, whole != 0, d_docs, ndocs, max_depth, d_out};
  int launched = 0;
  const bool good = ok(c, gram::launch_shard_edges(a, whole != 0, max_depth > 0xFFFFFFFFull ? 0xFFFFFFFFu : uint32_t(max_depth), failed, m->d_gram_scratch[i],
                                                    comm_target(m, st->seq, 0), xchg_gram_at(st->seq, uint32_t(m->rank)), st->stream, &launched),
                       "grammar edges");
  c->launches += unsigned(launched);
  return pass_end(m, good);
}

// Complete the oldest pass in flight, a grammar pass: round 0 (kind), the edge round and its fold (errors every rank sees
// alike, the halo, the bases), then pass A and the fold tree up with the record round, then the incoming stack, the
// fold tree down, pass C and the result round, whose fold gives the last document's result and the counts.
extern "C" int sjb200_document_errors_sharded_finish(sjb200_comm *m, sjb200_sharded_document_errors_result *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  memset(out, 0, sizeof(*out));
  out->error = SJB200_UNEXPECTED_ERROR;
  out->first_doc_in_error = out->first_error_index = UINT64_MAX;
  const uint32_t slot = m->tail % uint32_t(kXchgSteps);
  sjb200_comm::Step st;
  int rc = pass_pop(m, kGrammar, &st);
  if (rc != SJB200_SUCCESS) return rc;
  const sjb200_comm::GramStep gs = m->gram[slot];
  const int me = m->rank, R = m->nranks;
  if ((rc = comm_collect(m, st.seq, 4, kGramEdgeAt, kGramEdgeWords)) != SJB200_SUCCESS) return rc;
  sjb200_grammar_edge e[kMaxRanks];
  for (int r = 0; r < R; r++) {
    const unsigned long long *w = m->h_rec + size_t(r) * kGramWords + kGramEdgeAt;
    e[r] = sjb200_grammar_edge{uint32_t(w[0]), uint32_t(w[1]), uint32_t(w[2]), uint32_t(w[3]), uint32_t(w[4]), uint32_t(w[5])};
  }
  sjb200_grammar_edge_fold_result res;
  sjb200_grammar_rank ranks[kMaxRanks];
  int err = sjb200_grammar_edge_fold(R, e, &res, ranks);
  out->docs_before = ranks[me].docs_before;
  out->tokens_before = ranks[me].tokens_before;
  if (err != SJB200_SUCCESS) {
    int failed = -1;
    for (int r = 0; r < R && failed < 0; r++)
      if (e[r].flags & kGramEdgeFailed) failed = r;
    if (failed >= 0 && failed != me)
      c->last_error = "sharded grammar pass " + std::to_string(st.seq) + ": rank " + std::to_string(failed) + " could not run its pass";
    else if (failed < 0 && err == SJB200_UNEXPECTED_ERROR)
      c->last_error = "sharded grammar pass " + std::to_string(st.seq) + ": the ranks disagree on whole or max_depth";
    out->error = err;
    return err;
  }
  out->ndocs = res.ndocs;
  out->error = SJB200_SUCCESS;
  if (!gs.whole && res.ndocs == 0) return SJB200_SUCCESS;  // no document on any rank: nothing to judge
  cudaStream_t s = m->poll_stream;
  gram::ShardPass p{};
  p.a.type = gs.type; p.a.payload = gs.payload; p.a.n = gs.n;
  p.a.docs = gs.ndocs ? reinterpret_cast<const sjb200_doc_boundary_t *>(gs.docs) : nullptr;
  p.a.ndocs = gs.ndocs; p.a.max_depth = uint32_t(gs.max_depth);
  p.whole = gs.whole;
  p.owned = ranks[me].owned;
  p.tokens_before = ranks[me].tokens_before;
  p.out = reinterpret_cast<gram::sjb200_sharded_document_error_t *>(gs.out);
  if (res.bad_table) {  // every result {UNEXPECTED_ERROR, none}
    if (!ok(c, gram::launch_shard_fill_bad(p, s), "grammar results") || !ok(c, cudaStreamSynchronize(s), "sync")) return SJB200_UNEXPECTED_ERROR;
    c->launches += p.owned ? 1 : 0;
    c->last_error = "sharded grammar pass: a rank's document table is not strictly ascending or has an entry at or above its n";
    out->ndocs_in_error = res.ndocs;
    out->first_doc_in_error = res.ndocs ? 0 : UINT64_MAX;
    out->first_error = res.ndocs ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
    out->error = SJB200_UNEXPECTED_ERROR;
    return SJB200_UNEXPECTED_ERROR;
  }
  const gram::ShardHalo h{ranks[me].halo_before, ranks[me].halo_after, ranks[me].halo_flags, ranks[me].last_type};
  const Xchg x = comm_target(m, st.seq, 2);
  const size_t at = xchg_gram_at(st.seq, uint32_t(me));
  uint32_t *scratch = m->d_gram_scratch[slot];
  int launched = 0;
  // record round
  if (!ok(c, gram::launch_shard_records(p, h, ranks[me].holds_root != 0, scratch, c->sm_count, x, at, s, &launched), "grammar records"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += unsigned(launched);
  if ((rc = comm_collect(m, st.seq, 4, kGramRecAt, 2 + int((p.a.max_depth + 31) / 32))) != SJB200_SUCCESS) return rc;
  // result round
  if (!ok(c, gram::launch_shard_check(p, h, scratch, m->window + xchg_gram_at(st.seq, 0), c->sm_count, x, at, s, &launched), "grammar check"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += unsigned(launched);
  if ((rc = comm_collect(m, st.seq, 4, kGramResAt, kGramResWords)) != SJB200_SUCCESS) return rc;
  sjb200_grammar_tally t[kMaxRanks];
  for (int r = 0; r < R; r++) {
    const unsigned long long *w = m->h_rec + size_t(r) * kGramWords + kGramResAt;
    auto u64 = [&](int k) { return uint64_t(uint32_t(w[k])) | (uint64_t(uint32_t(w[k + 1])) << 32); };
    t[r] = sjb200_grammar_tally{u64(0), u64(2), u64(6), uint32_t(w[4]), uint32_t(w[5])};
  }
  sjb200_sharded_document_error last[kMaxRanks];
  err = sjb200_grammar_result_fold(R, e, t, out, last);
  out->docs_before = ranks[me].docs_before;
  out->tokens_before = ranks[me].tokens_before;
  if (p.owned && !ok(c, gram::launch_shard_store(p.out + (p.owned - 1), last[me].error, last[me].index, s), "grammar result")) return SJB200_UNEXPECTED_ERROR;
  c->launches += p.owned ? 1 : 0;
  if (!ok(c, cudaStreamSynchronize(s), "sync")) return SJB200_UNEXPECTED_ERROR;
  return err;
}

extern "C" int sjb200_document_errors_sharded(sjb200_comm *m, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, int whole,
                                              const sjb200_doc_boundary *d_docs, uint32_t ndocs, size_t max_depth, sjb200_sharded_document_error *d_out,
                                              sjb200_sharded_document_errors_result *out, void *stream) {
  int rc = sjb200_document_errors_sharded_enqueue(m, d_type, d_payload, n, whole, d_docs, ndocs, max_depth, d_out, stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_document_errors_sharded_finish(m, out);
}

// ---------------------------------------------------------------------------------------------- sharded JSON Pointer
namespace {
// FNV-1a over the compiled pointers: the ranks must walk the same ones
uint64_t blob_hash(const std::vector<uint8_t> &b) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (uint8_t c : b) h = (h ^ c) * 0x100000001b3ull;
  return h;
}

// wait (host polling, bounded) until `nwords` words from word `first` of every rank's part of the pass's pointer block
// (stride words apart) carry seq; the block's head (edge and count words) -> comm->h_rec
int ptr_collect(sjb200_comm *m, uint32_t seq, int first, int stride, int nwords) {
  sjb200_ctx *c = m->ctx;
  const unsigned long long *src = m->window + xchg_ptr_at(seq);
  const auto t0 = std::chrono::steady_clock::now();
  for (;;) {
    if (!ok(c, cudaMemcpyAsync(m->h_rec, src, size_t(kPtrHeadWords) * 8, cudaMemcpyDeviceToHost, m->poll_stream), "D2H window") ||
        !ok(c, cudaStreamSynchronize(m->poll_stream), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->xchg_polls++;
    bool all = true;
    for (int r = 0; r < m->nranks && all; r++)
      for (int k = 0; k < nwords; k++) all = all && uint32_t(m->h_rec[size_t(first) + size_t(r) * stride + k] >> 32) == seq;
    if (all) {
      c->xchg_wait_ms += ms_since(t0);
      return SJB200_SUCCESS;
    }
    if (std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - t0).count() > m->poll_timeout_ms) {
      c->last_error = "sharded pointer pass: a peer's words did not arrive";
      return SJB200_UNEXPECTED_ERROR;
    }
  }
}
}  // namespace

// Enqueue one pointer pass: the pointers compiled on the host into the slot's device blob, the first token in error of
// each document and of the leading segment, the table's check, then the edge words and the round-0 record into every
// rank's window.  The walks wait for finish, which knows where the documents end.  A rank that cannot run its pass (bad
// arguments, device allocation) or is over a limit still publishes, flagged, so that every rank's finish returns alike.
extern "C" int sjb200_at_pointer_sharded_enqueue(sjb200_comm *m, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                                 size_t string_bytes, int whole, const sjb200_doc_boundary *d_docs, uint32_t ndocs,
                                                 const char *const *pointers, const size_t *pointer_lens, int npointers,
                                                 sjb200_sharded_pointer_result *d_out, void *stream) {
  if (!m || !m->connected) return SJB200_UNEXPECTED_ERROR;
  sjb200_comm::Step *st = pass_begin(m, kPointer, 0, 0, nullptr, 0, nullptr, nullptr, stream);
  if (!st) return SJB200_CAPACITY;
  static_assert(sizeof(sjb200_sharded_pointer_result) == sizeof(ptr::ShardPtrResult), "layout");
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  const uint32_t i = m->head % uint32_t(kXchgSteps);
  if (whole || !d_docs) ndocs = 0;
  bool failed = npointers < 0 || (npointers && (!pointers || !pointer_lens)) || (n && (!d_type || !d_payload)) || (string_bytes && !d_strbuf) ||
                (npointers && !d_out && (whole ? m->rank == 0 : ndocs > 0));
  if (failed) c->last_error = "sharded pointer pass: bad arguments";
  bool over = npointers > kPtrMaxPointers;
  ptr::CompiledPointers cp;
  std::vector<uint8_t> blob;
  if (!failed && !over) {
    const int rc = ptr::compile_pointers(pointers, pointer_lens, npointers, &cp);
    over = rc == SJB200_CAPACITY;
    failed = rc != SJB200_SUCCESS && !over;
    if (failed) c->last_error = "sharded pointer pass: a null pointer with a non-zero length";
  }
  size_t hb = 0, lb = 0;
  if (!failed && !over) {
    hb = cp.headers.size() * sizeof(ptr::PtrHeader);
    lb = cp.levels.size() * sizeof(ptr::PtrLevel);
    blob.resize(hb + lb + cp.keys.size() + 1, 0);
    memcpy(blob.data(), cp.headers.data(), hb);
    memcpy(blob.data() + hb, cp.levels.data(), lb);
    memcpy(blob.data() + hb + lb, cp.keys.data(), cp.keys.size());
  }
  failed = failed || !grow(c, &m->d_ptr_scratch[i], &m->ptr_scratch_words[i], ptr::shard_scratch_words(ndocs), "cudaMalloc(pointer scratch)") ||
           (!blob.empty() && !grow(c, &m->d_ptr_blob[i], &m->ptr_blob_bytes[i], blob.size(), "cudaMalloc(pointers)"));
  ptr::PtrShard &s = m->ptrs[i].s;
  s = ptr::PtrShard{};
  m->ptrs[i].whole = whole != 0;
  const uint8_t *db = m->d_ptr_blob[i];
  s.a.w = ptr::Walk{d_type, d_payload, d_strbuf, string_bytes, reinterpret_cast<const ptr::PtrLevel *>(db + hb), db + hb + lb};
  s.a.n = n;
  s.a.docs = ndocs ? reinterpret_cast<const sjb200_doc_boundary_t *>(d_docs) : nullptr;
  s.a.ndocs = ndocs;
  s.a.headers = reinterpret_cast<const ptr::PtrHeader *>(db);
  s.a.npointers = uint32_t(npointers > 0 ? npointers : 0);
  s.out = reinterpret_cast<ptr::ShardPtrResult *>(d_out);
  s.scratch = m->d_ptr_scratch[i];
  const uint32_t flags = (failed ? uint32_t(kPtrEdgeFailed) : 0u) | (whole ? uint32_t(kPtrEdgeWhole) : 0u) | (over ? uint32_t(kPtrEdgeOver) : 0u);
  if (failed || over) s.a.npointers = 0;  // (nothing is walked: finish fails on every rank)
  bool good = blob.empty() || ok(c, cudaMemcpyAsync(m->d_ptr_blob[i], blob.data(), blob.size(), cudaMemcpyHostToDevice, st->stream), "H2D pointers");
  int launched = 0;
  good = good && ok(c, ptr::launch_shard_edges(s, flags, failed || over ? 0 : blob_hash(blob), comm_target(m, st->seq, 0), xchg_ptr_at(st->seq), c->sm_count,
                                               st->stream, &launched), "pointer edges");
  s.a.npointers = uint32_t(npointers > 0 && npointers <= kPtrMaxPointers ? npointers : 0);
  c->launches += unsigned(launched);
  return pass_end(m, good);
}

// Complete the oldest pass in flight, a pointer pass: round 0 (kind), the edge round and its fold (errors every rank
// sees alike, the bases, the holders, the tail documents), then the steps: the local walks, and while a step hands walks
// over, the next holders resume them.  Every step ends with a count round.  The results that came back from later ranks
// go into d_out last.
extern "C" int sjb200_at_pointer_sharded_finish(sjb200_comm *m, sjb200_sharded_pointer_summary *out) {
  if (!m || !out || m->tail == m->head) return SJB200_UNEXPECTED_ERROR;
  sjb200_ctx *c = m->ctx;
  DeviceGuard g(c->device);
  memset(out, 0, sizeof(*out));
  out->error = SJB200_UNEXPECTED_ERROR;
  const uint32_t slot = m->tail % uint32_t(kXchgSteps);
  sjb200_comm::Step st;
  int rc = pass_pop(m, kPointer, &st);
  if (rc != SJB200_SUCCESS) return rc;
  ptr::PtrShard s = m->ptrs[slot].s;
  const int me = m->rank, R = m->nranks;
  if ((rc = ptr_collect(m, st.seq, 0, kPtrEdgeWords, kPtrEdgeWords)) != SJB200_SUCCESS) return rc;
  sjb200_pointer_edge e[kMaxRanks];
  for (int r = 0; r < R; r++) {
    const unsigned long long *w = m->h_rec + size_t(r) * kPtrEdgeWords;
    auto u = [&](int k) { return uint32_t(w[k]); };
    e[r] = sjb200_pointer_edge{u(0), u(1), u(2), u(3), uint64_t(u(4)) | (uint64_t(u(5)) << 32), u(6), u(7), u(8), u(9)};
  }
  sjb200_pointer_edge_fold_result res;
  sjb200_pointer_rank ranks[kMaxRanks];
  int err = sjb200_pointer_edge_fold(R, e, &res, ranks);
  const sjb200_pointer_rank &k = ranks[me];
  out->docs_before = k.docs_before;
  out->tokens_before = k.tokens_before;
  out->ndocs = res.ndocs;
  cudaStream_t ps = m->poll_stream;
  if (err != SJB200_SUCCESS) {
    int failed = -1;
    for (int r = 0; r < R && failed < 0; r++)
      if (e[r].flags & kPtrEdgeFailed) failed = r;
    if (failed >= 0 && failed != me)
      c->last_error = "sharded pointer pass " + std::to_string(st.seq) + ": rank " + std::to_string(failed) + " could not run its pass";
    else if (failed < 0 && err == SJB200_UNEXPECTED_ERROR)
      c->last_error = "sharded pointer pass " + std::to_string(st.seq) + ": the ranks disagree on whole or on the pointers";
    out->error = err;
    return err;
  }
  s.tokens_before = k.tokens_before;
  s.owned = k.owned;
  const uint64_t np = s.a.npointers;
  if (res.bad_table || (m->ptrs[slot].whole && res.n == 0)) {  // every result {UNEXPECTED_ERROR, none}
    if (!ok(c, ptr::launch_shard_fill(s.out, np * s.owned, ptr::kUnexpectedError, c->sm_count, ps), "pointer results") || !ok(c, cudaStreamSynchronize(ps), "sync"))
      return SJB200_UNEXPECTED_ERROR;
    c->launches += (np && s.owned) ? 1 : 0;
    if (res.bad_table) c->last_error = "sharded pointer pass: a rank's document table is not strictly ascending or has an entry at or above its n";
    out->error = res.bad_table ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
    return out->error;
  }
  out->error = SJB200_SUCCESS;
  if ((!m->ptrs[slot].whole && res.ndocs == 0) || np == 0) return SJB200_SUCCESS;  // no document on any rank / no pointer
  const size_t base = xchg_ptr_at(st.seq);
  auto area = [&](int r, size_t at) { return r < 0 ? nullptr : m->peer[r] + base + at; };
  s.v = ptr::ShardView{s.a.n, k.next_type, k.tail_continues, uint64_t(s.a.n) + k.tail_after};
  s.walks = k.walks;
  s.lead_end = e[me].first_entry;
  s.tail_err = int32_t(k.tail_error);
  s.tail_err_index = k.tail_error_index;
  s.tail_res = k.tail_owner >= 0 && k.tail_owner != me ? area(k.tail_owner, kPtrResAt) : nullptr;
  s.lead_res = k.lead_owner >= 0 && k.lead_owner != me ? area(k.lead_owner, kPtrResAt) : nullptr;
  s.seq = st.seq;
  const Xchg x = comm_target(m, st.seq, 2);
  // step 0: the local walks; step t > 0: the walks handed over in step t - 1.  A rank writes step t's records into the
  // next holder's buffer t % 2 only after every rank's count of step t - 1 arrived, and the reader of buffer t % 2
  // (step t - 2's records) posted that count after its resume: the buffers never overlap in time.
  uint32_t step = 0;
  for (;; step++) {
    s.step = step;
    s.next_rec = area(k.next_holder, kPtrRecAt + size_t(step & 1u) * kPtrMaxPointers * 2);
    s.rec_in = m->window + base + kPtrRecAt + size_t((step + 1) & 1u) * kPtrMaxPointers * 2;
    int launched = 0;
    if (step == 0) {
      if (!ok(c, ptr::launch_shard_walks(s, c->sm_count, ps, &launched), "pointer walks")) return SJB200_UNEXPECTED_ERROR;
    } else if (k.prev_holder >= 0 && uint32_t(m->h_rec[kPtrCountAt + size_t(k.prev_holder) * kMaxRanks + step - 1]) > 0) {
      const bool cta = s.lead_end > ptr::kCtaMinStructurals;  // (the piece the walks resume over)
      if (!ok(c, ptr::launch_shard_resume(s, cta, ps), "pointer resume")) return SJB200_UNEXPECTED_ERROR;
      launched = 1;
    }
    if (!ok(c, ptr::launch_shard_post_count(s.scratch, x, base, step, ps), "pointer count")) return SJB200_UNEXPECTED_ERROR;
    c->launches += unsigned(launched) + 1;
    if ((rc = ptr_collect(m, st.seq, kPtrCountAt + int(step), kMaxRanks, 1)) != SJB200_SUCCESS) return rc;
    uint64_t handed = 0;
    for (int r = 0; r < R; r++) handed += uint32_t(m->h_rec[kPtrCountAt + size_t(r) * kMaxRanks + step]);
    out->walks_forwarded += uint32_t(m->h_rec[kPtrCountAt + size_t(me) * kMaxRanks + step]);
    if (handed == 0) break;
    if (step + 1 >= uint32_t(R)) {  // (a walk crosses each cut at most once)
      c->last_error = "sharded pointer pass: walks still handed over after every rank";
      return SJB200_UNEXPECTED_ERROR;
    }
  }
  out->rounds = step;
  // the results of this rank's document that ended on later ranks
  const bool gets = s.owned && (m->ptrs[slot].whole ? k.walks == 0 || k.tail_continues : (k.tail_owner == me && k.tail_continues));
  if (gets && !ok(c, ptr::launch_shard_scatter(m->window + base + kPtrResAt, st.seq, s.out, uint32_t(np), s.owned, ps), "pointer results"))
    return SJB200_UNEXPECTED_ERROR;
  c->launches += gets ? 1 : 0;
  if (!ok(c, cudaStreamSynchronize(ps), "sync")) return SJB200_UNEXPECTED_ERROR;
  return SJB200_SUCCESS;
}

extern "C" int sjb200_at_pointer_sharded(sjb200_comm *m, const uint8_t *d_type, const uint64_t *d_payload, uint32_t n, const uint8_t *d_strbuf,
                                         size_t string_bytes, int whole, const sjb200_doc_boundary *d_docs, uint32_t ndocs, const char *const *pointers,
                                         const size_t *pointer_lens, int npointers, sjb200_sharded_pointer_result *d_out,
                                         sjb200_sharded_pointer_summary *out, void *stream) {
  int rc = sjb200_at_pointer_sharded_enqueue(m, d_type, d_payload, n, d_strbuf, string_bytes, whole, d_docs, ndocs, pointers, pointer_lens, npointers, d_out,
                                             stream);
  if (rc != SJB200_SUCCESS) return rc;
  return sjb200_at_pointer_sharded_finish(m, out);
}
