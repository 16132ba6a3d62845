// grammar_shards_emul.cpp -- the sharded stage-2 grammar pass (sjb200_document_errors_sharded) under the host SIMT
// emulation: every rank's share of the pass runs the tile routines of simdjson_b200/csrc/sjb200_grammar.cuh with its
// ShardHalo, and the pure host folds of simdjson_b200/csrc/sjb200_fold.cpp run between the rounds, with the exchange
// windows in host memory.  The rounds, in the order the ranks' finish runs them:
//   edges    shard_edge_words per rank -> sjb200_grammar_edge_fold (the halo, the bases, the verdicts every rank shares)
//   records  per rank: the start bitmap (table, and bit 0 on the rank that holds the stream's structural 0), pass A with
//            the halo, the fold tree up; the top record into the window
//   results  per rank: shard_incoming from the window, the fold tree down, pass C (errors into each document's slot or
//            the leading slot), the results of all documents but the last, shard_result_words -> sjb200_grammar_result_fold
// 32 OS threads are the lanes of one warp (sjb200_simt.cuh, SJB200_HOST_EMU).  Tiles of 32 x ITEMS structurals, ITEMS 1,
// 2 or 32.  Driven by tests/test_document_errors_shards_emul.py; no GPU involved.
#define SJB200_HOST_EMU 1
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include <functional>
#include <vector>

#include "../include/sjb200.h"
#include "sjb200_grammar.cuh"

using namespace sjb200;
thread_local simt::ThreadCtx simt::tctx;

namespace {

// run fn(lane) on the 32 lanes of one emulated warp
struct Warp {
  std::function<void(unsigned)> fn;
  simt::CtaShared cta;
  simt::WarpShared warp;
};
struct LaneArg { Warp *w; unsigned lane; };
void *lane_main(void *vp) {
  LaneArg *a = static_cast<LaneArg *>(vp);
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->lane;
  simt::tctx.nctas = 1;
  simt::tctx.warp = &a->w->warp;
  simt::tctx.ctas = &a->w->cta;
  a->w->fn(a->lane);
  return nullptr;
}
bool run_warp(const std::function<void(unsigned)> &fn) {
  Warp w;
  w.fn = fn;
  pthread_barrier_init(&w.warp.bar, nullptr, 32);
  pthread_barrier_init(&w.cta.bar, nullptr, 32);
  w.cta.smem = nullptr;
  std::vector<LaneArg> args(32);
  std::vector<pthread_t> th(32);
  bool good = true;
  for (unsigned t = 0; t < 32; t++) {
    args[t] = LaneArg{&w, t};
    if (pthread_create(&th[t], nullptr, lane_main, &args[t]) != 0) good = false;
  }
  for (unsigned t = 0; t < 32; t++) pthread_join(th[t], nullptr);
  pthread_barrier_destroy(&w.warp.bar);
  pthread_barrier_destroy(&w.cta.bar);
  return good;
}

struct Rank {
  const uint8_t *type;
  const uint64_t *payload;
  uint32_t n;
  std::vector<uint32_t> docs;           // the rank's table, local
  std::vector<uint32_t> starts;         // start bitmap
  std::vector<uint32_t> records;        // fold tree levels, then the incoming record
  std::vector<size_t> level_at;
  std::vector<uint32_t> level_count;
  std::vector<unsigned long long> first;
  gram::ShardHalo halo;
  uint32_t owned;
  uint64_t tokens_before;
};

template <int ITEMS>
void pass_records(Rank &k, const gram::Grammar &g0, std::vector<uint8_t> &smem) {
  run_warp([&](unsigned lane) {
    gram::TileSmem<ITEMS> &sm = *reinterpret_cast<gram::TileSmem<ITEMS> *>(smem.data());
    const gram::Grammar g = g0;
    const uint32_t kTile = gram::TileSmem<ITEMS>::kTile, tiles = (g.n + kTile - 1) / kTile;
    const size_t stride = 2 + g.words;
    uint32_t *rec = k.records.data();
    for (uint32_t t = 0; t < tiles; t++) {
      gram::load_tile<ITEMS>(g, sm, lane, t * kTile, k.halo);
      gram::tile_record<ITEMS>(g, sm, lane, t * kTile, rec + k.level_at[0] * stride + size_t(t) * stride, k.halo);
    }
    for (size_t l = 0; l + 1 < k.level_count.size(); l++)
      for (uint32_t gr = 0; gr < (k.level_count[l] + 31) / 32; gr++)
        gram::fold_up_group(lane, sm.rec, sm.child, rec + k.level_at[l] * stride, k.level_count[l], rec + k.level_at[l + 1] * stride, gr, g.words);
  });
}

template <int ITEMS>
void pass_check(Rank &k, const gram::Grammar &g0, std::vector<uint8_t> &smem, const std::vector<std::vector<uint32_t>> &window, uint32_t rank, bool whole) {
  run_warp([&](unsigned lane) {
    gram::TileSmem<ITEMS> &sm = *reinterpret_cast<gram::TileSmem<ITEMS> *>(smem.data());
    gram::Grammar g = g0;
    const uint32_t kTile = gram::TileSmem<ITEMS>::kTile, tiles = (g.n + kTile - 1) / kTile;
    const size_t stride = 2 + g.words, L = k.level_count.size();
    uint32_t *rec = k.records.data();
    uint32_t *incoming = rec + k.level_at[L] * stride;
    gram::shard_incoming(lane, sm.rec, sm.child, [&](uint32_t r, uint32_t w) { return window[r][w]; }, rank, g.words, incoming);
    for (size_t l = L; l-- > 0;)
      for (uint32_t gr = 0; gr < (k.level_count[l] + 31) / 32; gr++)
        gram::fold_down_group(lane, sm.rec, sm.child, rec + k.level_at[l] * stride, k.level_count[l],
                              l + 1 < L ? rec + k.level_at[l + 1] * stride : incoming, gr, g.words);
    g.prefix = rec;
    auto report = [&](uint32_t pos, uint32_t code, uint32_t index) {
      uint32_t d = gram::kNone;
      if (!whole) {
        uint32_t lo = 0, hi = uint32_t(k.docs.size());
        while (lo < hi) {
          const uint32_t mid = lo + (hi - lo) / 2;
          if (k.docs[mid] <= pos) lo = mid + 1; else hi = mid;
        }
        d = lo == 0 ? gram::kNone : lo - 1;
      }
      unsigned long long *slot = &k.first[gram::shard_slot(whole, d, k.owned)];
      const unsigned long long key = (static_cast<unsigned long long>(index) << 8) | code;
      unsigned long long cur = __atomic_load_n(slot, __ATOMIC_SEQ_CST);
      while (key < cur && !__atomic_compare_exchange_n(slot, &cur, key, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
      }
    };
    for (uint32_t t = 0; t < tiles; t++) {
      gram::load_tile<ITEMS>(g, sm, lane, t * kTile, k.halo);
      gram::tile_check<ITEMS>(g, sm, lane, t * kTile, t, report, k.halo);
    }
  });
}

}  // namespace

// One stream of n structurals (types / payloads, a table of nstarts ascending starts or whole = 1 for one document) cut
// into nranks shards at the token cuts[0..nranks] (cuts[0] = 0, cuts[nranks] = n), through the sharded pass.  Writes the
// gathered results (errors / indexes, one per document) and summary[6] = {finish's error, ndocs, ndocs_in_error,
// first_doc_in_error, first_error, first_error_index}.  Returns 0, or -1 for bad arguments.
extern "C" int emu_sharded_document_errors(int items, int nranks, const uint8_t *type, const uint64_t *payload, const uint32_t *cuts, int whole,
                                           const uint32_t *starts, uint32_t nstarts, uint32_t max_depth, int32_t *errors, uint64_t *indexes,
                                           uint64_t *summary) {
  if ((items != 1 && items != 2 && items != 32) || nranks < 1 || nranks > kMaxRanks) return -1;
  const uint32_t md = max_depth == 0 ? 1u : max_depth > gram::kMaxDepth ? gram::kMaxDepth : max_depth;
  const uint32_t words = (md + 31) / 32;
  std::vector<Rank> ranks(static_cast<size_t>(nranks));
  sjb200_grammar_edge e[kMaxRanks];
  for (int r = 0; r < nranks; r++) {
    Rank &k = ranks[size_t(r)];
    k.type = type + cuts[r];
    k.payload = payload + cuts[r];
    k.n = cuts[r + 1] - cuts[r];
    for (uint32_t j = 0; !whole && j < nstarts; j++)
      if (starts[j] >= cuts[r] && starts[j] < cuts[r + 1]) k.docs.push_back(starts[j] - cuts[r]);
    uint32_t w[kGramEdgeWords];
    const uint32_t nd = uint32_t(k.docs.size());
    bool bad = false;
    for (uint32_t j = 1; j < nd; j++) bad = bad || k.docs[j] <= k.docs[j - 1];
    gram::shard_edge_words(k.type, k.n, whole != 0, nd, nd ? k.docs[0] : 0u, nd ? k.docs[nd - 1] : 0u, bad, false, max_depth, w);
    e[r] = sjb200_grammar_edge{w[0], w[1], w[2], w[3], w[4], w[5]};
  }
  // edge round
  sjb200_grammar_edge_fold_result res;
  sjb200_grammar_rank rk[kMaxRanks];
  const int err = sjb200_grammar_edge_fold(nranks, e, &res, rk);
  memset(summary, 0, 6 * sizeof(uint64_t));
  summary[0] = uint64_t(err);
  if (err != SJB200_SUCCESS || res.bad_table || (!whole && res.ndocs == 0)) {
    summary[0] = res.bad_table && err == SJB200_SUCCESS ? uint64_t(SJB200_UNEXPECTED_ERROR) : summary[0];
    summary[1] = err == SJB200_SUCCESS ? res.ndocs : 0;
    return 0;
  }
  std::vector<uint8_t> smem(sizeof(gram::TileSmem<32>));
  std::vector<std::vector<uint32_t>> window(size_t(nranks), std::vector<uint32_t>(2 + words, 0));
  std::vector<gram::Grammar> gs(static_cast<size_t>(nranks));
  const uint32_t tile = 32u * uint32_t(items);
  // record round
  for (int r = 0; r < nranks; r++) {
    Rank &k = ranks[size_t(r)];
    k.halo = gram::ShardHalo{rk[r].halo_before, rk[r].halo_after, rk[r].halo_flags, rk[r].last_type};
    k.owned = rk[r].owned;
    k.tokens_before = rk[r].tokens_before;
    k.starts.assign((k.n + 31) / 32 + 1, 0);
    for (uint32_t s : k.docs) k.starts[s >> 5] |= 1u << (s & 31u);
    if (rk[r].holds_root) k.starts[0] |= 1u;
    for (uint32_t c = (k.n + tile - 1) / tile;; c = (c + 31) / 32) {
      k.level_count.push_back(c);
      if (c <= 1) break;
    }
    size_t at = 0;
    for (uint32_t c : k.level_count) {
      k.level_at.push_back(at);
      at += c;
    }
    k.level_at.push_back(at);  // the incoming record
    k.records.assign((at + 1) * (2 + words), 0xA5A5A5A5u);
    k.first.assign(k.owned + 1, ~0ull);
    gram::Grammar &g = gs[size_t(r)];
    g.type = k.type; g.payload = k.payload; g.n = k.n; g.starts = k.starts.data(); g.whole = whole != 0;
    g.max_depth = md; g.words = words; g.prefix = nullptr;
    if (k.n) {
      if (items == 1) pass_records<1>(k, g, smem);
      else if (items == 2) pass_records<2>(k, g, smem);
      else pass_records<32>(k, g, smem);
      const uint32_t *top = k.records.data() + k.level_at[k.level_count.size() - 1] * (2 + words);
      for (uint32_t w = 0; w < 2 + words; w++) window[size_t(r)][w] = (w < 2 || w - 2 < (top[1] + 31) / 32) ? top[w] : 0u;
    }
  }
  // result round
  sjb200_grammar_tally t[kMaxRanks];
  for (int r = 0; r < nranks; r++) {
    Rank &k = ranks[size_t(r)];
    if (k.n) {
      if (items == 1) pass_check<1>(k, gs[size_t(r)], smem, window, uint32_t(r), whole != 0);
      else if (items == 2) pass_check<2>(k, gs[size_t(r)], smem, window, uint32_t(r), whole != 0);
      else pass_check<32>(k, gs[size_t(r)], smem, window, uint32_t(r), whole != 0);
    }
    uint32_t errs = 0, fd = gram::kNone;
    for (uint32_t d = 0; d + 1 < k.owned; d++) {
      int32_t er;
      uint64_t ix;
      gram::shard_doc_result(k.first[d], k.tokens_before, k.docs[d + 1], &er, &ix);
      errors[rk[r].docs_before + d] = er;
      indexes[rk[r].docs_before + d] = ix;
      if (er) {
        errs++;
        if (fd == gram::kNone) fd = d;
      }
    }
    uint32_t w[kGramResWords];
    gram::shard_result_words(k.first.data(), k.owned, k.tokens_before, errs, fd, w);
    t[r] = sjb200_grammar_tally{uint64_t(w[0]) | uint64_t(w[1]) << 32, uint64_t(w[2]) | uint64_t(w[3]) << 32, uint64_t(w[6]) | uint64_t(w[7]) << 32, w[4], w[5]};
  }
  sjb200_sharded_document_errors_result out;
  sjb200_sharded_document_error last[kMaxRanks];
  sjb200_grammar_result_fold(nranks, e, t, &out, last);
  for (int r = 0; r < nranks; r++)
    if (rk[r].owned) {
      errors[rk[r].docs_before + rk[r].owned - 1] = last[r].error;
      indexes[rk[r].docs_before + rk[r].owned - 1] = last[r].index;
    }
  summary[0] = uint64_t(out.error);
  summary[1] = out.ndocs;
  summary[2] = out.ndocs_in_error;
  summary[3] = out.first_doc_in_error;
  summary[4] = uint64_t(uint32_t(out.first_error));
  summary[5] = out.first_error_index;
  return 0;
}
