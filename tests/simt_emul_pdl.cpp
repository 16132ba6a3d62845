// simt_emul_pdl.cpp -- consecutive multi-document launches of the ACTUAL scan4 kernel source (sjb200_scan4.cuh) that
// overlap the way programmatic dependent launch lets them overlap on the GPU, under the host SIMT emulation
// (sjb200_simt.cuh, SJB200_HOST_EMU).  Launch k + 1 starts once every CTA of launch k has triggered or exited;
// sj_griddep_wait blocks until every thread of the previous launch has exited.  The launches share the context's
// scratch the way the host code does: ticket block, launch flags word and look-back descriptors in two sets, chosen by
// launch parity, every document its own carry and flags word.  Checked against the oracle: every document's carry and
// flags, and the index arrays the launches share (they must hold what the last writer wrote).  Test infrastructure only.
//
// build: see tests/test_simt_emul_pdl.py
#define SJB200_HOST_EMU 1
#include "sjb200_scan4.cuh"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

extern "C" {
#include "sj_oracle.h"
}

using namespace sjb200;

thread_local simt::ThreadCtx simt::tctx;

namespace {

// one emulated grid: its threads, barriers and shared memory, and its dependency state
struct Grid {
  unsigned nctas = 0;
  ScanParams p;
  std::vector<simt::CtaShared> ctas;
  std::vector<simt::WarpShared> warps;
  std::unique_ptr<std::atomic<unsigned>[]> cta_alive;
  std::unique_ptr<std::atomic<uint8_t>[]> cta_released;
  simt::GridDep dep;
  std::vector<pthread_t> th;
};
struct ThreadArg {
  Grid *g;
  unsigned tid, ctaid;
};

void *thread_main(void *arg) {
  ThreadArg *a = static_cast<ThreadArg *>(arg);
  Grid *g = a->g;
  const unsigned W = unsigned(scan4::kThreads4) / 32;
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->tid;
  simt::tctx.cta = a->ctaid;
  simt::tctx.nctas = g->nctas;
  simt::tctx.warp = &g->warps[a->ctaid * W + a->tid / 32];
  simt::tctx.ctas = &g->ctas[a->ctaid];
  simt::tctx.dep = &g->dep;
  sj_tensor_map unused{};
  scan4::scan4_body<0>(&unused, g->p, g->ctas[a->ctaid].smem, uint32_t(reinterpret_cast<uintptr_t>(g->ctas[a->ctaid].smem)));
  if (g->cta_alive[a->ctaid].fetch_sub(1) == 1) sj_griddep_launch_dependents();  // the CTA's exit counts as its trigger
  g->dep.running.fetch_sub(1, std::memory_order_release);
  return nullptr;
}

// Runs the launches as a chain: launch k + 1's threads are created once launch k has released every CTA.
void emu_chain(std::vector<std::unique_ptr<Grid>> &grids) {
  const unsigned T = unsigned(scan4::kThreads4), W = T / 32;
  const size_t smem_bytes = size_t(scan4::kSmemBytes4);
  std::vector<std::vector<ThreadArg>> args(grids.size());
  pthread_attr_t attr;
  pthread_attr_init(&attr);
  pthread_attr_setstacksize(&attr, 256 * 1024);
  for (size_t k = 0; k < grids.size(); k++) {
    Grid &g = *grids[k];
    if (k > 0) {
      while (grids[k - 1]->dep.released.load() != grids[k - 1]->nctas) {
        struct timespec ts = {0, 50000};
        nanosleep(&ts, nullptr);
      }
      g.dep.prev = &grids[k - 1]->dep;
    }
    g.ctas.resize(g.nctas);
    g.warps = std::vector<simt::WarpShared>(size_t(g.nctas) * W);
    g.cta_alive.reset(new std::atomic<unsigned>[g.nctas]);
    g.cta_released.reset(new std::atomic<uint8_t>[g.nctas]);
    g.dep.cta_released = g.cta_released.get();
    g.dep.running = g.nctas * T;
    for (unsigned c = 0; c < g.nctas; c++) {
      g.cta_alive[c] = T;
      g.cta_released[c] = 0;
      pthread_barrier_init(&g.ctas[c].bar, nullptr, T);
      g.ctas[c].smem = static_cast<uint8_t *>(aligned_alloc(1024, (smem_bytes + 1023) & ~size_t(1023)));
      memset(g.ctas[c].smem, 0xCD, smem_bytes);
      for (unsigned w = 0; w < W; w++) pthread_barrier_init(&g.warps[c * W + w].bar, nullptr, 32);
    }
    args[k].resize(size_t(g.nctas) * T);
    g.th.resize(size_t(g.nctas) * T);
    for (unsigned c = 0; c < g.nctas; c++)
      for (unsigned t = 0; t < T; t++) {
        ThreadArg &a = args[k][size_t(c) * T + t];
        a.g = &g; a.tid = t; a.ctaid = c;
        if (pthread_create(&g.th[size_t(c) * T + t], &attr, thread_main, &a) != 0) { perror("pthread_create"); exit(3); }
      }
  }
  for (auto &g : grids) {
    for (auto &t : g->th) pthread_join(t, nullptr);
    for (unsigned c = 0; c < g->nctas; c++) {
      free(g->ctas[c].smem);
      pthread_barrier_destroy(&g->ctas[c].bar);
      for (unsigned w = 0; w < W; w++) pthread_barrier_destroy(&g->warps[c * W + w].bar);
    }
  }
  pthread_attr_destroy(&attr);
}

std::vector<uint8_t> random_doc(std::mt19937_64 &rng, bool tiny) {
  const char *alpha = "\\\"\" {}[],: \n\tabc1\x01\xc3\xa9";
  const size_t sizes[] = {1, 3, 100, 4095, 4096, 4097, 65535, 65536, 65537, 70000, 140000};
  size_t n = tiny ? 1 + rng() % 200 : sizes[rng() % 11] + rng() % 3;
  std::vector<uint8_t> d;
  for (size_t i = 0; i < n; i++) d.push_back(uint8_t(rng() % 4 ? 'a' + rng() % 26 : alpha[rng() % strlen(alpha)]));
  return d;
}

struct Doc {
  std::vector<uint8_t> store;  // the input, 16-byte aligned (or `misalign` bytes past it)
  const uint8_t *buf = nullptr;
  size_t len = 0;
  int out = 0;                 // index array it writes
  int in_from = -1;            // >= 0: its input is bytes [in_off, in_off + len) of the index array this document of the previous launch writes
  size_t in_off = 0;
};

int g_fail = 0;

// launches[k] = the documents of launch k, which write nout index arrays.  A launch with a document that reads an index
// array has early_input 0.
void check_chain(std::vector<std::vector<Doc>> &launches, int nout, unsigned max_grid, std::mt19937_64 &rng, uint32_t *epoch, const char *what) {
  size_t max_len = 1;
  for (auto &L : launches)
    for (auto &d : L) max_len = std::max(max_len, d.len);
  std::vector<std::vector<uint32_t>> outs(size_t(nout), std::vector<uint32_t>(max_len + 16, 0xABABABABu));
  size_t ndocs = 0;
  for (auto &L : launches) ndocs += L.size();
  std::vector<Carry> carry(ndocs);
  std::vector<uint32_t> docflags(ndocs, 0);
  uint32_t ticket[2][4] = {};
  uint32_t lflags[2] = {0, 0};
  size_t max_elems = 1;
  for (auto &L : launches) {
    size_t e = 0;
    for (auto &d : L) e += (d.len + scan4::kElemBytes - 1) / scan4::kElemBytes;
    max_elems = std::max(max_elems, e);
  }
  std::vector<unsigned long long> desc[2] = {std::vector<unsigned long long>(max_elems + 1, 0ull), std::vector<unsigned long long>(max_elems + 1, 0ull)};
  std::vector<std::vector<DocEntry>> tabs(launches.size());
  std::vector<std::vector<sj_tensor_map>> maps(launches.size());
  std::vector<std::unique_ptr<Grid>> grids;
  size_t slot = 0;
  std::vector<std::vector<size_t>> slots(launches.size());
  for (size_t k = 0; k < launches.size(); k++) {
    auto &L = launches[k];
    tabs[k].resize(L.size());
    maps[k].resize(L.size());
    uint32_t elems = 0, tiles = 0;
    bool early = true;
    for (size_t i = 0; i < L.size(); i++) {
      Doc &d = L[i];
      if (d.in_from >= 0) {
        d.buf = reinterpret_cast<const uint8_t *>(outs[size_t(launches[k - 1][size_t(d.in_from)].out)].data()) + d.in_off;
        early = false;
      }
      maps[k][i].base = d.buf; maps[k][i].rows = d.len / 128; maps[k][i].box_rows = scan4::kBlockRows;
      DocEntry &e = tabs[k][i];
      e.buf = d.buf;
      e.idx_out = outs[size_t(d.out)].data();
      e.carry_out = &carry[slot];
      e.carry_out_host = nullptr;
      e.flags = &docflags[slot];
      e.tmap = ((reinterpret_cast<uintptr_t>(d.buf) & 15u) == 0 && maps[k][i].rows > 0) ? &maps[k][i] : nullptr;
      e.len = uint32_t(d.len);
      e.scan_end = e.len;
      e.first_elem = elems;
      e.nelem = uint32_t((d.len + scan4::kElemBytes - 1) / scan4::kElemBytes);
      elems += e.nelem;
      tiles += uint32_t((d.len + kTileBytes - 1) / kTileBytes);
      slots[k].push_back(slot++);
    }
    const int parity = int(k & 1);
    grids.emplace_back(new Grid());
    Grid &g = *grids.back();
    g.nctas = std::min<unsigned>(1 + unsigned(rng() % max_grid), elems);
    ScanParams &p = g.p;
    memset(&p, 0, sizeof(p));
    p.prev_word = 0x20202020u; p.check_eof = 1; p.write_sentinels = 1; p.epoch = ++*epoch; p.ntiles = tiles;
    p.flags = &lflags[parity]; p.count_desc = desc[parity].data(); p.ticket = ticket[parity];
    p.docs = tabs[k].data(); p.ndocs = uint32_t(L.size());
    p.early_input = early ? 1u : 0u;
  }
  emu_chain(grids);
  if (lflags[0] || lflags[1]) { fprintf(stderr, "BUG: launch flags not re-armed (%s)\n", what); g_fail++; }
  for (int q = 0; q < 2; q++)
    if (ticket[q][0] || ticket[q][1] || ticket[q][2]) { fprintf(stderr, "BUG: ticket block %d not re-armed (%s)\n", q, what); g_fail++; }
  for (uint32_t f : docflags)
    if (f) { fprintf(stderr, "BUG: document flags not handed over (%s)\n", what); g_fail++; break; }
  // the oracle, launch by launch: a document that reads an index array sees its content after the previous launch
  const size_t nb = size_t(nout);
  std::vector<std::vector<uint32_t>> want_out(nb), prev_words(nb);
  std::vector<int> last_writer(nb, -1);
  for (size_t k = 0; k < launches.size(); k++) {
    std::vector<std::vector<uint32_t>> now = prev_words;
    for (size_t i = 0; i < launches[k].size(); i++) {
      const Doc &d = launches[k][i];
      std::vector<uint8_t> in(d.len);
      if (d.in_from >= 0) {
        const std::vector<uint32_t> &w = prev_words[size_t(launches[k - 1][size_t(d.in_from)].out)];
        if (w.size() * 4 < d.in_off + d.len) { fprintf(stderr, "harness: input beyond the words it reads\n"); exit(2); }
        memcpy(in.data(), reinterpret_cast<const uint8_t *>(w.data()) + d.in_off, d.len);
      } else {
        memcpy(in.data(), d.buf, d.len);
      }
      std::vector<uint32_t> oidx(d.len + 16);
      uint32_t ostate = 0;
      const uint64_t on = sjo_scan_shard(in.data(), d.len, 0, oidx.data(), &ostate);
      oidx[on] = uint32_t(d.len); oidx[on + 1] = uint32_t(d.len); oidx[on + 2] = 0;
      oidx.resize(on + 3);
      const Carry &r = carry[slots[k][i]];
      int bad = 0;
      if (r.flags & kFlagInternal) bad = 1;
      else if (r.count != on) bad = 2;
      else if ((r.state & 7u) != (ostate & 7u)) bad = 5;
      else if (bool(r.flags & kFlagUtf8) == bool(sjo_validate_utf8(in.data(), d.len))) bad = 6;
      else if (r.ttable != sjo_transducer(in.data(), d.len)) bad = 7;
      if (bad) {
        fprintf(stderr, "MISMATCH kind=%d (%s) launch %zu doc %zu len=%zu in_from=%d: got n=%llu state=%u flags=%u | want n=%llu state=%u\n", bad, what, k, i,
                d.len, d.in_from, (unsigned long long)r.count, r.state, r.flags, (unsigned long long)on, ostate);
        g_fail++;
      }
      // what the document leaves in its index array: its words over what was there
      std::vector<uint32_t> &o = now[size_t(d.out)];
      if (o.size() < oidx.size()) o.resize(oidx.size(), 0xABABABABu);
      memcpy(o.data(), oidx.data(), oidx.size() * 4);
      want_out[size_t(d.out)] = o;
      last_writer[size_t(d.out)] = int(k);
    }
    prev_words = now;
  }
  for (int b = 0; b < nout; b++) {
    const std::vector<uint32_t> &w = want_out[size_t(b)];
    if (w.empty()) continue;
    if (memcmp(outs[size_t(b)].data(), w.data(), w.size() * 4) != 0) {
      size_t at = 0;
      while (outs[size_t(b)][at] == w[at]) at++;
      fprintf(stderr, "MISMATCH (%s) index array %d (last written by launch %d): word %zu got %u want %u\n", what, b, last_writer[size_t(b)], at,
              outs[size_t(b)][at], w[at]);
      g_fail++;
    }
  }
}

Doc make_doc(std::vector<uint8_t> bytes, int out, size_t misalign) {
  Doc d;
  d.store.assign(bytes.size() + misalign + 16, 0);
  memcpy(d.store.data() + misalign, bytes.data(), bytes.size());
  d.buf = d.store.data() + misalign;
  d.len = bytes.size();
  d.out = out;
  return d;
}

}  // namespace

int main(int argc, char **argv) {
  const int iters = argc > 1 ? atoi(argv[1]) : 6;
  std::mt19937_64 rng(0x9D1);
  uint32_t epoch = 0;
  for (int it = 0; it < iters && g_fail < 5; it++) {
    // four index arrays that every launch writes again (a batch over 4 rotating buffers); half the iterations with
    // documents of at most 200 bytes, one element each: every launch's descriptors start at element 0
    const bool tiny = (it & 1) != 0;
    const size_t nl = 3 + rng() % 3;
    std::vector<std::vector<Doc>> launches(nl);
    for (auto &L : launches)
      for (int b = 0; b < 4; b++) L.push_back(make_doc(random_doc(rng, tiny), b, rng() % 4 == 0 ? 1 + rng() % 15 : 0));
    check_chain(launches, 4, 3, rng, &epoch, tiny ? "tiny documents, 4 shared index arrays" : "4 shared index arrays");
  }
  {
    // launch k + 1 reads what launch k wrote (early_input 0): its second document is the end of the index array the
    // previous launch's first document writes (the words its last elements and its sentinels leave there)
    std::vector<std::vector<Doc>> launches(4);
    std::vector<uint8_t> rows;
    while (rows.size() < 12 * size_t(scan4::kElemBytes) + 77) {
      const char *row = "{\"k\": [1, \"v\\\"\", true]},\n";
      rows.insert(rows.end(), row, row + strlen(row));
    }
    std::vector<uint32_t> ridx(rows.size() + 16);
    uint32_t rstate = 0;
    const size_t rn = size_t(sjo_scan_shard(rows.data(), rows.size(), 0, ridx.data(), &rstate));
    for (size_t k = 0; k < launches.size(); k++) {
      const int base = int(2 * k);  // fresh index arrays per launch
      if (k == 0) {
        launches[k].push_back(make_doc(rows, base, 0));
        launches[k].push_back(make_doc(random_doc(rng, false), base + 1, 0));
      } else {  // the dependent document first: its elements are the launch's first tickets
        Doc d;
        d.len = 4096 + 1000 * k;
        d.in_off = (4 * (rn + 3) - d.len) & ~size_t(15);
        d.out = base + 1;
        d.in_from = k == 1 ? 0 : 1;
        launches[k].push_back(d);
        launches[k].push_back(make_doc(rows, base, 0));
      }
    }
    check_chain(launches, 8, 3, rng, &epoch, "input written by the previous launch");
  }
  if (g_fail) { printf("FAILED\n"); return 1; }
  printf("simt emulation of overlapped launches OK (%d cases)\n", iters + 1);
  return 0;
}
