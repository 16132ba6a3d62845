// grammar_emul.cpp -- the stage-2 grammar pass (simdjson_b200/csrc/sjb200_grammar.cuh) under the host SIMT emulation:
// 32 OS threads are the lanes of one warp, which runs every tile of pass A, the fold tree of pass B and every tile of
// pass C in turn (sjb200_simt.cuh, SJB200_HOST_EMU).  Tiles of 32 x ITEMS structurals, ITEMS 1, 2 or 32, so that small
// inputs span many tiles.  Driven by tests/test_document_errors_emul.py against the oracle; no GPU involved.
#define SJB200_HOST_EMU 1
#include <pthread.h>
#include <stdint.h>

#include <vector>

#include "sjb200_grammar.cuh"

using namespace sjb200;
thread_local simt::ThreadCtx simt::tctx;

namespace {

struct Job {
  gram::Grammar g;
  const uint32_t *docs;
  uint32_t ndocs;
  std::vector<uint32_t> *records;  // every level of the fold tree, then the identity
  std::vector<size_t> level_at;    // record offset of each level
  std::vector<uint32_t> level_count;
  std::vector<unsigned long long> first;
  simt::CtaShared cta;
  simt::WarpShared warp;
  void *smem;
};

template <int ITEMS>
void *thread_main(Job *j, unsigned lane) {
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = lane;
  simt::tctx.nctas = 1;
  simt::tctx.warp = &j->warp;
  simt::tctx.ctas = &j->cta;
  gram::TileSmem<ITEMS> &sm = *static_cast<gram::TileSmem<ITEMS> *>(j->smem);
  gram::Grammar g = j->g;
  const uint32_t kTile = gram::TileSmem<ITEMS>::kTile;
  const uint32_t tiles = (g.n + kTile - 1) / kTile;
  const size_t stride = 2 + g.words;
  uint32_t *rec = j->records->data();
  for (uint32_t t = 0; t < tiles; t++) {
    gram::load_tile<ITEMS>(g, sm, lane, t * kTile);
    gram::tile_record<ITEMS>(g, sm, lane, t * kTile, rec + j->level_at[0] * stride + size_t(t) * stride);
  }
  const size_t L = j->level_count.size();
  for (size_t l = 0; l + 1 < L; l++)
    for (uint32_t gr = 0; gr < (j->level_count[l] + 31) / 32; gr++)
      gram::fold_up_group(lane, sm.rec, sm.child, rec + j->level_at[l] * stride, j->level_count[l], rec + j->level_at[l + 1] * stride, gr, g.words);
  for (size_t l = L; l-- > 0;)
    for (uint32_t gr = 0; gr < (j->level_count[l] + 31) / 32; gr++)
      gram::fold_down_group(lane, sm.rec, sm.child, rec + j->level_at[l] * stride, j->level_count[l],
                            rec + (l + 1 < L ? j->level_at[l + 1] : j->level_at[L]) * stride, gr, g.words);
  g.prefix = rec;
  auto report = [&](uint32_t pos, uint32_t code, uint32_t index) {
    uint32_t d = 0;
    if (j->docs) {
      uint32_t lo = 0, hi = j->ndocs;
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (j->docs[mid] <= pos) lo = mid + 1; else hi = mid;
      }
      if (lo == 0) return;
      d = lo - 1;
    }
    const unsigned long long key = (static_cast<unsigned long long>(index) << 8) | code;
    unsigned long long cur = __atomic_load_n(&j->first[d], __ATOMIC_SEQ_CST);
    while (key < cur && !__atomic_compare_exchange_n(&j->first[d], &cur, key, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
    }
  };
  for (uint32_t t = 0; t < tiles; t++) {
    gram::load_tile<ITEMS>(g, sm, lane, t * kTile);
    gram::tile_check<ITEMS>(g, sm, lane, t * kTile, t, report);
  }
  return nullptr;
}

struct Arg { Job *job; unsigned lane; int items; };
void *entry(void *vp) {
  Arg *a = static_cast<Arg *>(vp);
  if (a->items == 1) return thread_main<1>(a->job, a->lane);
  if (a->items == 2) return thread_main<2>(a->job, a->lane);
  return thread_main<32>(a->job, a->lane);
}

}  // namespace

// Every document of the stream (docs: ndocs ascending starts below n, or null for one document [0, n)) through the three
// passes; errors / indexes as sjb200_document_errors_dev writes them for a valid table and n > 0.  Returns 0, or -1.
extern "C" int emu_document_errors(int items, const uint8_t *type, const uint64_t *payload, uint32_t n, const uint32_t *docs, uint32_t ndocs,
                                   uint32_t max_depth, int32_t *errors, uint32_t *indexes) {
  if (n == 0 || (items != 1 && items != 2 && items != 32)) return -1;
  Job job;
  job.g.type = type;
  job.g.payload = payload;
  job.g.n = n;
  job.g.whole = docs == nullptr;
  job.g.max_depth = max_depth;
  job.g.words = (max_depth + 31) / 32;
  job.docs = docs;
  job.ndocs = docs ? ndocs : 1;
  std::vector<uint32_t> starts((n + 31) / 32 + 1, 0);
  starts[0] = 1;
  for (uint32_t d = 0; docs && d < ndocs; d++) starts[docs[d] >> 5] |= 1u << (docs[d] & 31u);
  job.g.starts = starts.data();
  const uint32_t tile = 32u * uint32_t(items);
  for (uint32_t c = (n + tile - 1) / tile;; c = (c + 31) / 32) {
    job.level_count.push_back(c);
    if (c <= 1) break;
  }
  size_t at = 0;
  for (uint32_t c : job.level_count) {
    job.level_at.push_back(at);
    at += c;
  }
  job.level_at.push_back(at);  // the identity
  std::vector<uint32_t> records((at + 1) * (2 + job.g.words), 0xA5A5A5A5u);
  for (uint32_t w = 0; w < 2 + job.g.words; w++) records[at * (2 + job.g.words) + w] = 0;
  job.records = &records;
  job.first.assign(job.ndocs, ~0ull);
  std::vector<uint8_t> smem(sizeof(gram::TileSmem<32>));
  job.smem = smem.data();
  pthread_barrier_init(&job.warp.bar, nullptr, 32);
  pthread_barrier_init(&job.cta.bar, nullptr, 32);
  job.cta.smem = nullptr;
  std::vector<Arg> args(32);
  std::vector<pthread_t> th(32);
  for (unsigned t = 0; t < 32; t++) {
    args[t] = Arg{&job, t, items};
    if (pthread_create(&th[t], nullptr, entry, &args[t]) != 0) return -1;
  }
  for (auto &t : th) pthread_join(t, nullptr);
  pthread_barrier_destroy(&job.warp.bar);
  pthread_barrier_destroy(&job.cta.bar);
  for (uint32_t d = 0; d < job.ndocs; d++) {
    if (job.first[d] != ~0ull) {
      errors[d] = int32_t(job.first[d] & 0xFF);
      indexes[d] = uint32_t(job.first[d] >> 8);
    } else {
      errors[d] = 0;
      indexes[d] = docs && d + 1 < ndocs ? docs[d + 1] : n;
    }
  }
  return 0;
}
