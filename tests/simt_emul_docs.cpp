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

#include "simt_fenced.h"

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

// one launch over `docs`; misalign[k] != 0: the document starts that many bytes past a 16-byte boundary (plain loads).
// packed: the documents are consecutive, gapless pieces of one buffer (NDJSON rows in memory: a neighbour ends in a
// backslash, inside a string, on a UTF-8 lead byte), and their index arrays are consecutive pieces of exactly
// sjb200_index_words(len) words of another; both buffers end at an inaccessible page (the input starts right after one
// when in_at_end is false), so a read outside the documents or a write outside the index arrays kills the process, and
// the words of each array past its structurals and sentinels must still hold their fill
void check_launch(std::vector<std::vector<uint8_t>> &docs, const std::vector<size_t> &misalign, unsigned grid, uint32_t epoch, const char *what,
                  bool packed = false, bool in_at_end = true) {
  const size_t n = docs.size();
  std::vector<std::vector<uint8_t>> store(n);
  std::vector<std::vector<uint32_t>> idx(n);
  std::vector<uint32_t *> ip(n);
  std::vector<size_t> nwords(n);
  size_t in_bytes = 0, out_words = 0;
  for (size_t k = 0; k < n; k++) in_bytes += docs[k].size(), out_words += index_words(docs[k].size());
  Fenced in(packed ? in_bytes : 0, in_at_end), out(packed ? out_words * 4 : 0, true);
  size_t in_off = 0, out_off = 0;
  std::vector<sj_tensor_map> maps(n);
  std::vector<DocEntry> tab(n);
  std::vector<Carry> carry(n);
  std::vector<uint32_t> flags(n + 1, 0);
  uint32_t elems = 0;
  for (size_t k = 0; k < n; k++) {
    const uint8_t *buf;
    if (packed) {
      memcpy(in.p + in_off, docs[k].data(), docs[k].size());
      buf = in.p + in_off;
      in_off += docs[k].size();
      nwords[k] = index_words(docs[k].size());
      ip[k] = reinterpret_cast<uint32_t *>(out.p) + out_off;
      out_off += nwords[k];
      for (size_t i = 0; i < nwords[k]; i++) ip[k][i] = 0xABABABABu;
    } else {
      store[k].assign(docs[k].size() + misalign[k] + 16, 0);
      memcpy(store[k].data() + misalign[k], docs[k].data(), docs[k].size());
      buf = store[k].data() + misalign[k];
      idx[k].assign(docs[k].size() + 16, 0xABABABABu);
      ip[k] = idx[k].data();
      nwords[k] = idx[k].size();
    }
    maps[k].base = buf; maps[k].rows = docs[k].size() / 128; maps[k].box_rows = scan4::kBlockRows;
    DocEntry &e = tab[k];
    e.buf = buf;
    e.idx_out = ip[k];
    e.carry_out = &carry[k];
    e.carry_out_host = nullptr;
    e.flags = &flags[1 + k];
    e.tmap = (misalign[k] == 0 && (reinterpret_cast<uintptr_t>(buf) & 15u) == 0 && maps[k].rows > 0) ? &maps[k] : nullptr;
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
    else if (memcmp(ip[k], oidx.data(), on * 4) != 0) bad = 3;
    else if (ip[k][on] != uint32_t(len) || ip[k][on + 1] != uint32_t(len) || ip[k][on + 2] != 0) bad = 4;
    else if ((r.state & 7u) != (ostate & 7u)) bad = 5;
    else if (bool(r.flags & kFlagUtf8) == bool(sjo_validate_utf8(buf, len))) bad = 6;
    else if (r.ttable != sjo_transducer(buf, len)) bad = 7;
    for (size_t i = on + 3; i < nwords[k] && !bad; i++)
      if (ip[k][i] != 0xABABABABu) bad = 8;  // a word past the structurals and sentinels
    if (bad) {
      fprintf(stderr, "MISMATCH kind=%d (%s) doc %zu of %zu len=%zu misalign=%zu packed=%d grid=%u: got n=%llu state=%u flags=%u | want n=%llu state=%u\n", bad, what, k,
              n, len, misalign[k], int(packed), grid, (unsigned long long)r.count, r.state, r.flags, (unsigned long long)on, ostate);
      g_fail++;
    }
  }
}

}  // namespace

// the packed, fenced launches: documents whose ends are hostile to a neighbour that reads across them
int run_fenced(std::mt19937_64 &rng, uint32_t &epoch) {
  static const char *tails[] = {"\\", "\"ab", "\xf0\x9f\x98", "\xc3", "12", "tru", "\\\\\\"};
  static const char heads[] = {'\x80', '"', '\\', '7'};
  for (int it = 0; it < 24 && g_fail < 5; it++) {
    const size_t n = 2 + rng() % 7;
    std::vector<std::vector<uint8_t>> docs;
    for (size_t k = 0; k < n; k++) {
      std::vector<uint8_t> d = random_doc(rng);
      d[0] = uint8_t(heads[rng() % 4]);
      const char *t = tails[rng() % 7];
      const size_t tl = std::min(strlen(t), d.size());
      memcpy(d.data() + d.size() - tl, t + strlen(t) - tl, tl);
      docs.push_back(d);
    }
    check_launch(docs, std::vector<size_t>(n, 0), 1 + unsigned(rng() % 3), ++epoch, "packed, fenced", true, it % 2 == 0);
  }
  return g_fail;
}

int main(int argc, char **argv) {
  std::mt19937_64 rng(0xD0C5);
  uint32_t epoch = 0;
  if (argc > 1 && strcmp(argv[1], "--fenced") == 0) {
    if (run_fenced(rng, epoch)) { printf("FAILED\n"); return 1; }
    printf("simt emulation of packed, fenced multi-document launches OK\n");
    return 0;
  }
  const int iters = argc > 1 ? atoi(argv[1]) : 24;
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
