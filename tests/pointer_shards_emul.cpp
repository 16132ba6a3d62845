// pointer_shards_emul.cpp -- the sharded JSON Pointer pass (sjb200_at_pointer_sharded) under the host SIMT emulation:
// every rank's walks (walk_from of simdjson_b200/csrc/sjb200_pointer.cuh with the rank's ShardCut, by a warp group or a
// CTA group of OS threads), with the pure edge fold (sjb200_pointer_edge_fold, sjb200_fold.cpp) between the rounds and
// the continuation records (pack_walk / unpack_walk) handed from rank to rank as the window carries them.  Driven by
// tests/test_pointer_shards_emul.py against the oracle and the unsharded emulation; no GPU involved.
#define SJB200_HOST_EMU 1
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../include/sjb200.h"
#include "sjb200_params.h"
#include "sjb200_pointer.cuh"

using namespace sjb200;
thread_local simt::ThreadCtx simt::tctx;

namespace {
constexpr unsigned kCtaWarps = 8;  // the sm_90a build's CTA group (sjb200_pointer.h)
constexpr int kCtaItems = 8;

struct Task {  // one walk of a step
  uint32_t p;
  ptr::WalkAt at;
  uint32_t end;
  // out
  uint32_t v;
  int32_t err;
  ptr::WalkAt susp;
};

struct Group {
  ptr::Walk w;
  const ptr::PtrHeader *headers;
  ptr::ShardView view;
  std::vector<Task> *tasks;
  ptr::CtaSmem<kCtaWarps> sm;
  simt::CtaShared cta;
  std::vector<simt::WarpShared> warps;
};
struct ThreadArg { Group *g; unsigned tid; bool cta; };

void *thread_main(void *vp) {
  ThreadArg *a = static_cast<ThreadArg *>(vp);
  Group &j = *a->g;
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->tid;
  simt::tctx.nctas = 1;
  simt::tctx.warp = &j.warps[a->tid / 32];
  simt::tctx.ctas = &j.cta;
  ptr::WarpGroup wg{a->tid & 31u};
  ptr::CtaGroup<kCtaWarps> cg{a->tid, &j.sm};
  for (Task &t : *j.tasks) {
    int32_t e;
    ptr::WalkAt s{};
    const ptr::ShardCut cut = ptr::piece_cut(j.view, t.end);
    const uint32_t v = a->cta ? ptr::walk_from<ptr::CtaGroup<kCtaWarps>, kCtaItems>(cg, j.w, j.headers[t.p], t.at, t.end, cut, &e, &s)
                              : ptr::walk_from<ptr::WarpGroup, 1>(wg, j.w, j.headers[t.p], t.at, t.end, cut, &e, &s);
    if (a->tid == 0) {
      t.v = v;
      t.err = e;
      t.susp = s;
    }
  }
  return nullptr;
}

// run the tasks of one rank's step on one group of threads
int run_group(bool cta, const ptr::Walk &w, const ptr::PtrHeader *headers, const ptr::ShardView &view, std::vector<Task> *tasks) {
  if (tasks->empty()) return 0;
  Group g;
  g.w = w;
  g.headers = headers;
  g.view = view;
  g.tasks = tasks;
  const unsigned T = cta ? 32 * kCtaWarps : 32;
  g.warps.resize(T / 32);
  for (auto &x : g.warps) pthread_barrier_init(&x.bar, nullptr, 32);
  pthread_barrier_init(&g.cta.bar, nullptr, T);
  g.cta.smem = nullptr;
  std::vector<ThreadArg> args(T);
  std::vector<pthread_t> th(T);
  for (unsigned t = 0; t < T; t++) {
    args[t] = ThreadArg{&g, t, cta};
    if (pthread_create(&th[t], nullptr, thread_main, &args[t]) != 0) return -1;
  }
  for (auto &t : th) pthread_join(t, nullptr);
  for (auto &x : g.warps) pthread_barrier_destroy(&x.bar);
  pthread_barrier_destroy(&g.cta.bar);
  return 0;
}
}  // namespace

// The gathered tokens (type, payload, strbuf) cut into nranks shards at token cuts[0..nranks] (cuts[0] = 0, cuts[nranks]
// = n) and string-buffer cuts sbase[0..nranks]; every rank gets its own copy with rank-local string payloads, exactly
// as sjb200_tokens_sharded leaves them.  whole = 1: one document; else the document starts (global structural indexes,
// ascending) split into the ranks' tables.  Pointer k: the next lens[k] bytes of `pointers`.  err / idx: [np][D] with
// D = 1 (whole) or nstarts, the gathered results (UINT64_MAX: none); stats: [0] continuation steps, [1] walks handed
// over, [2] the fold's error.  Returns compile_pointers' code, or -1.
extern "C" int emu_sharded_at_pointer(int cta, int nranks, const uint8_t *type, const uint64_t *payload, const uint8_t *strbuf, const uint32_t *cuts,
                                      const uint64_t *sbase, int whole, const uint32_t *starts, uint32_t nstarts, const char *pointers, const size_t *lens,
                                      int np, int32_t *err, uint64_t *idx, uint64_t *stats) {
  if (nranks < 1 || nranks > kMaxRanks) return -1;
  std::vector<const char *> ptrs(size_t(np > 0 ? np : 1));
  for (int k = 0; k < np; k++) {
    ptrs[size_t(k)] = pointers;
    pointers += lens[k];
  }
  ptr::CompiledPointers cp;
  const int rc = ptr::compile_pointers(ptrs.data(), lens, np, &cp);
  if (rc != 0) return rc;
  const uint32_t D = whole ? 1u : nstarts;
  for (size_t i = 0; i < size_t(np) * D; i++) {
    err[i] = -1;
    idx[i] = 0;
  }
  // the ranks' inputs and edges
  std::vector<std::vector<uint8_t>> rt(static_cast<size_t>(nranks)), rs(static_cast<size_t>(nranks));
  std::vector<std::vector<uint64_t>> rp(static_cast<size_t>(nranks));
  std::vector<std::vector<uint32_t>> table(static_cast<size_t>(nranks));
  sjb200_pointer_edge e[kMaxRanks];
  for (int r = 0; r < nranks; r++) {
    const uint32_t b = cuts[r], n = cuts[r + 1] - cuts[r];
    rt[r].assign(type + b, type + b + n);
    rp[r].assign(payload + b, payload + b + n);
    for (uint32_t k = 0; k < n; k++)
      if (rt[r][k] == '"') rp[r][k] -= sbase[r];
    rs[r].assign(strbuf + sbase[r], strbuf + sbase[r + 1]);
    if (!whole)
      for (uint32_t d = 0; d < nstarts; d++)
        if (starts[d] >= b && starts[d] < b + n) table[r].push_back(starts[d] - b);
    const uint32_t lead_end = table[r].empty() ? n : table[r][0];
    uint32_t lead = 0xFFFFFFFFu;
    for (uint32_t k = 0; k < lead_end && lead == 0xFFFFFFFFu; k++)
      if (rt[r][k] == 0) lead = k;
    e[r] = sjb200_pointer_edge{n, uint32_t(table[r].size()), whole ? uint32_t(kPtrEdgeWhole) : 0u, uint32_t(np), 0,
                               n ? uint32_t(rt[r][0]) | (uint32_t(rt[r][n - 1]) << 8) : 0xFFFFu, lead_end, lead,
                               lead == 0xFFFFFFFFu ? 0u : uint32_t(rp[r][lead] & 0xFFu)};
  }
  sjb200_pointer_edge_fold_result res;
  sjb200_pointer_rank ranks[kMaxRanks];
  stats[2] = uint64_t(sjb200_pointer_edge_fold(nranks, e, &res, ranks));
  if (res.error != SJB200_SUCCESS) return 0;
  auto put = [&](uint32_t p, uint64_t gdoc, int32_t er, uint64_t ix) {
    err[size_t(p) * D + gdoc] = er;
    idx[size_t(p) * D + gdoc] = ix;
  };
  if ((!whole && res.ndocs == 0) || np == 0) return 0;
  if (whole && res.n == 0) {
    for (int p = 0; p < np; p++) put(uint32_t(p), 0, ptr::kUnexpectedError, ~0ull);
    return 0;
  }
  // the document of rank r's last structural / of its leading segment, as a global document number
  auto last_doc = [&](int owner) { return whole ? 0ull : ranks[owner].docs_before + ranks[owner].owned - 1; };
  std::vector<std::vector<Task>> inbox(static_cast<size_t>(nranks));  // the records handed to each rank in the previous step
  uint64_t forwarded = 0;
  uint32_t step = 0;
  for (;; step++) {
    std::vector<std::vector<Task>> next(static_cast<size_t>(nranks));
    uint64_t handed = 0;
    for (int r = 0; r < nranks; r++) {
      const sjb200_pointer_rank &k = ranks[r];
      const uint32_t n = e[r].n;
      const ptr::Walk w{rt[r].data(), rp[r].data(), rs[r].data(), rs[r].size(), cp.levels.data(), reinterpret_cast<const uint8_t *>(cp.keys.data())};
      const ptr::ShardView view{n, k.next_type, k.tail_continues, uint64_t(n) + k.tail_after};
      std::vector<Task> tasks;
      std::vector<uint64_t> gdoc;
      if (step == 0 && k.walks) {
        const uint32_t Dr = whole ? 1u : uint32_t(table[r].size());
        for (uint32_t d = 0; d < Dr; d++) {
          const uint32_t b = whole ? 0 : table[r][d], end = (whole || d + 1 == Dr) ? n : table[r][d + 1];
          const uint64_t g = whole ? 0 : k.docs_before + d;
          uint32_t fe = 0xFFFFFFFFu;
          for (uint32_t q = b; q < end && fe == 0xFFFFFFFFu; q++)
            if (rt[r][q] == 0) fe = q;
          for (int p = 0; p < np; p++) {
            if (fe != 0xFFFFFFFFu) {
              put(uint32_t(p), g, int32_t(rp[r][fe]), k.tokens_before + fe);
            } else if (end == n && k.tail_error) {
              put(uint32_t(p), g, int32_t(k.tail_error), k.tail_error_index);
            } else {
              tasks.push_back(Task{uint32_t(p), ptr::WalkAt{0, b, 0, 0, 0, 0}, end, 0, 0, {}});
              gdoc.push_back(g);
            }
          }
        }
      } else if (step > 0) {
        for (Task &t : inbox[r]) {
          tasks.push_back(Task{t.p, t.at, e[r].first_entry, 0, 0, {}});
          gdoc.push_back(last_doc(k.lead_owner));
        }
      }
      if (run_group(cta != 0, w, cp.headers.data(), view, &tasks) != 0) return -1;
      for (size_t i = 0; i < tasks.size(); i++) {
        const Task &t = tasks[i];
        if (t.v == ptr::kSuspend) {
          // through the 16-byte record, as the window carries it
          unsigned long long w0, w1;
          ptr::pack_walk(t.susp, 7, step, &w0, &w1);
          ptr::WalkAt back;
          if (k.next_holder < 0 || !ptr::unpack_walk(w0, w1, 7, step, &back)) return -1;
          next[size_t(k.next_holder)].push_back(Task{t.p, back, 0, 0, 0, {}});
          handed++;
          continue;
        }
        put(t.p, gdoc[i], t.err, t.v == ptr::kNone ? ~0ull : k.tokens_before + t.v);
      }
    }
    forwarded += handed;
    if (handed == 0) break;
    if (step + 1 >= uint32_t(nranks)) return -1;
    inbox.swap(next);
  }
  stats[0] = step;
  stats[1] = forwarded;
  return 0;
}
