// simt_emul_docs.cpp -- a multi-document launch of the ACTUAL scan4 kernel source (sjb200_scan4.cuh) under the host SIMT
// emulation (sjb200_simt.cuh, SJB200_HOST_EMU), checked document by document against the oracle.  Tickets and
// look-back descriptors run over the concatenation of the documents; a document that starts while the previous one is
// inside a string must not inherit that state (the look-back window stops at the document's first element, whose
// descriptor is an inclusive prefix from a zero state).  Test infrastructure only.
//
// build: see tests/test_simt_emul_docs.py
#define SJB200_HOST_EMU 1
#include "sjb200_scan4.cuh"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

extern "C" {
#include "sj_oracle.h"
}

using namespace sjb200;

thread_local simt::ThreadCtx simt::tctx;

namespace {

struct ThreadArg {
  const ScanParams *p;
  simt::CtaShared *cta;
  simt::WarpShared *warp;
  unsigned tid, ctaid, grid;
};
void *thread_main(void *arg) {
  ThreadArg *a = static_cast<ThreadArg *>(arg);
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->tid;
  simt::tctx.cta = a->ctaid;
  simt::tctx.nctas = a->grid;
  simt::tctx.warp = a->warp;
  simt::tctx.ctas = a->cta;
  sj_tensor_map unused{};
  scan4::scan4_body<0>(&unused, *a->p, a->cta->smem, uint32_t(reinterpret_cast<uintptr_t>(a->cta->smem)));
  return nullptr;
}

void emu_launch(unsigned grid, const ScanParams &p) {
  const unsigned T = unsigned(scan4::kThreads4), W = T / 32;
  const size_t smem_bytes = size_t(scan4::kSmemBytes4);
  std::vector<simt::CtaShared> ctas(grid);
  std::vector<simt::WarpShared> warps(size_t(grid) * W);
  std::vector<ThreadArg> args(size_t(grid) * T);
  std::vector<pthread_t> th(size_t(grid) * T);
  for (unsigned c = 0; c < grid; c++) {
    pthread_barrier_init(&ctas[c].bar, nullptr, T);
    ctas[c].smem = static_cast<uint8_t *>(aligned_alloc(1024, (smem_bytes + 1023) & ~size_t(1023)));
    memset(ctas[c].smem, 0xCD, smem_bytes);
    for (unsigned w = 0; w < W; w++) pthread_barrier_init(&warps[c * W + w].bar, nullptr, 32);
  }
  pthread_attr_t attr;
  pthread_attr_init(&attr);
  pthread_attr_setstacksize(&attr, 256 * 1024);
  for (unsigned c = 0; c < grid; c++)
    for (unsigned t = 0; t < T; t++) {
      ThreadArg &a = args[size_t(c) * T + t];
      a.p = &p; a.cta = &ctas[c]; a.warp = &warps[c * W + t / 32]; a.tid = t; a.ctaid = c; a.grid = grid;
      if (pthread_create(&th[size_t(c) * T + t], &attr, thread_main, &a) != 0) { perror("pthread_create"); exit(3); }
    }
  for (auto &t : th) pthread_join(t, nullptr);
  pthread_attr_destroy(&attr);
  for (unsigned c = 0; c < grid; c++) {
    free(ctas[c].smem);
    pthread_barrier_destroy(&ctas[c].bar);
    for (unsigned w = 0; w < W; w++) pthread_barrier_destroy(&warps[c * W + w].bar);
  }
}

std::vector<uint8_t> random_doc(std::mt19937_64 &rng) {
  const char *alpha = "\\\"\" {}[],: \n\tabc1\x01\xc3\xa9";
  const size_t sizes[] = {1, 3, 100, 4095, 4096, 4097, 65535, 65536, 65537, 70000, 140000};
  size_t n = sizes[rng() % 11] + rng() % 3;
  std::vector<uint8_t> d;
  for (size_t i = 0; i < n; i++) d.push_back(uint8_t(rng() % 4 ? 'a' + rng() % 26 : alpha[rng() % strlen(alpha)]));
  return d;
}

int g_fail = 0;

// one launch over `docs`; misalign[k] != 0: the document starts that many bytes past a 16-byte boundary (plain loads)
void check_launch(std::vector<std::vector<uint8_t>> &docs, const std::vector<size_t> &misalign, unsigned grid, uint32_t epoch, const char *what) {
  const size_t n = docs.size();
  std::vector<std::vector<uint8_t>> store(n);
  std::vector<std::vector<uint32_t>> idx(n);
  std::vector<sj_tensor_map> maps(n);
  std::vector<DocEntry> tab(n);
  std::vector<Carry> carry(n);
  std::vector<uint32_t> flags(n + 1, 0);
  uint32_t elems = 0;
  for (size_t k = 0; k < n; k++) {
    store[k].assign(docs[k].size() + misalign[k] + 16, 0);
    memcpy(store[k].data() + misalign[k], docs[k].data(), docs[k].size());
    const uint8_t *buf = store[k].data() + misalign[k];
    idx[k].assign(docs[k].size() + 16, 0xABABABABu);
    maps[k].base = buf; maps[k].rows = docs[k].size() / 128; maps[k].box_rows = scan4::kBlockRows;
    DocEntry &e = tab[k];
    e.buf = buf;
    e.idx_out = idx[k].data();
    e.carry_out = &carry[k];
    e.carry_out_host = nullptr;
    e.flags = &flags[1 + k];
    e.tmap = (misalign[k] == 0 && maps[k].rows > 0) ? &maps[k] : nullptr;
    e.len = uint32_t(docs[k].size());
    e.scan_end = e.len;
    e.first_elem = elems;
    e.nelem = uint32_t((docs[k].size() + scan4::kElemBytes - 1) / scan4::kElemBytes);
    elems += e.nelem;
  }
  std::vector<unsigned long long> desc(elems + 1, 0ull);
  uint32_t ticket[4] = {0, 0, 0, 0};
  ScanParams p;
  memset(&p, 0, sizeof(p));
  p.prev_word = 0x20202020u; p.check_eof = 1; p.write_sentinels = 1; p.epoch = epoch;
  p.flags = &flags[0]; p.count_desc = desc.data(); p.ticket = ticket;
  p.docs = tab.data(); p.ndocs = uint32_t(n);
  emu_launch(std::min<unsigned>(grid, elems), p);
  for (size_t i = 0; i <= n; i++)
    if (flags[i] != 0 || ticket[0] || ticket[1] || ticket[2]) { fprintf(stderr, "BUG: ticket/flags not re-armed (%s)\n", what); g_fail++; return; }
  for (size_t k = 0; k < n; k++) {
    const uint8_t *buf = tab[k].buf;
    const size_t len = docs[k].size();
    std::vector<uint32_t> oidx(len + 16);
    uint32_t ostate = 0;
    const uint64_t on = sjo_scan_shard(buf, len, 0, oidx.data(), &ostate);
    const Carry &r = carry[k];
    int bad = 0;
    if (r.flags & kFlagInternal) bad = 1;
    else if (r.count != on) bad = 2;
    else if (memcmp(idx[k].data(), oidx.data(), on * 4) != 0) bad = 3;
    else if (idx[k][on] != uint32_t(len) || idx[k][on + 1] != uint32_t(len) || idx[k][on + 2] != 0) bad = 4;
    else if ((r.state & 7u) != (ostate & 7u)) bad = 5;
    else if (bool(r.flags & kFlagUtf8) == bool(sjo_validate_utf8(buf, len))) bad = 6;
    else if (r.ttable != sjo_transducer(buf, len)) bad = 7;
    if (bad) {
      fprintf(stderr, "MISMATCH kind=%d (%s) doc %zu of %zu len=%zu misalign=%zu grid=%u: got n=%llu state=%u flags=%u | want n=%llu state=%u\n", bad, what, k, n, len,
              misalign[k], grid, (unsigned long long)r.count, r.state, r.flags, (unsigned long long)on, ostate);
      g_fail++;
    }
  }
}

}  // namespace

int main(int argc, char **argv) {
  const int iters = argc > 1 ? atoi(argv[1]) : 24;
  std::mt19937_64 rng(0xD0C5);
  uint32_t epoch = 0;
  // a document that ends inside a string, then a multi-element one: the later elements' look-back windows reach across
  // the boundary into descriptors of the same epoch
  {
    std::vector<std::vector<uint8_t>> docs;
    std::vector<uint8_t> a(70000, 'x');
    a[0] = '[';
    a[1] = '"';  // the string never closes
    docs.push_back(a);
    std::vector<uint8_t> b;
    while (b.size() < 5 * size_t(scan4::kElemBytes) + 77) {
      const char *row = "{\"k\": [1, \"v\\\"\", true]},\n";
      b.insert(b.end(), row, row + strlen(row));
    }
    docs.push_back(b);
    docs.push_back(std::vector<uint8_t>(1, '"'));
    docs.push_back(b);
    for (unsigned grid : {1u, 2u, 3u}) check_launch(docs, {0, 0, 0, 3}, grid, ++epoch, "string across the boundary");
  }
  for (int it = 0; it < iters && g_fail < 5; it++) {
    const size_t n = 2 + rng() % 6;
    std::vector<std::vector<uint8_t>> docs;
    std::vector<size_t> mis;
    for (size_t k = 0; k < n; k++) {
      docs.push_back(random_doc(rng));
      mis.push_back(rng() % 3 == 0 ? 1 + rng() % 15 : 0);
    }
    check_launch(docs, mis, 1 + unsigned(rng() % 3), ++epoch, "random");
  }
  if (g_fail) { printf("FAILED\n"); return 1; }
  printf("simt emulation of multi-document launches OK (%d cases)\n", iters);
  return 0;
}
