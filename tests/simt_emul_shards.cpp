// simt_emul_shards.cpp -- the per-shard launches of sharded minify / validate_utf8 / stage 1, from the ACTUAL kernel
// sources (sjb200_scan4.cuh, sjb200_utf8.cuh) under the host SIMT emulation (sjb200_simt.cuh, SJB200_HOST_EMU), with the
// exchange windows of every rank in host memory.  Checked against the oracle:
//   - the record each launch's last CTA stores into every rank's window: seq, kind, count, outgoing state, transducer,
//     flags (speculative launches, incoming state 0);
//   - minify launches with a non-zero carry-in (what a rank whose speculation failed runs): their kept bytes, placed at
//     the rank's base, give the oracle's minify of the whole buffer, cut at arbitrary bytes -- just after a backslash,
//     inside strings, inside UTF-8 characters;
//   - utf8v2's record for valid and corrupted shards cut at character boundaries.
// The fold of the records (sjb200_comm.cu) is host code and is not run here.  Test infrastructure only.
//
// build: see tests/test_simt_emul_shards.py
#define SJB200_HOST_EMU 1
#include "sjb200_scan4.cuh"
#include "sjb200_utf8.cuh"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

extern "C" {
#include "sj_oracle.h"
}

using namespace sjb200;

thread_local simt::ThreadCtx simt::tctx;

namespace {

// ------------------------------------------------------------------ launches (one OS thread per CUDA thread)
struct LaunchArgs {
  unsigned grid;
  const sj_tensor_map *tmap;
  const ScanParams *p;
  int mode;  // 0 stage 1, 2 minify, 3 validate_utf8 (utf8v2)
};
struct ThreadArg {
  const LaunchArgs *la;
  simt::CtaShared *cta;
  simt::WarpShared *warp;
  unsigned tid, ctaid;
};
void *thread_main(void *arg) {
  ThreadArg *a = static_cast<ThreadArg *>(arg);
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->tid;
  simt::tctx.cta = a->ctaid;
  simt::tctx.nctas = a->la->grid;
  simt::tctx.warp = a->warp;
  simt::tctx.ctas = a->cta;
  const uint32_t sa = uint32_t(reinterpret_cast<uintptr_t>(a->cta->smem));
  if (a->la->mode == 3) utf8v2::utf8_body(a->la->tmap, *a->la->p, a->cta->smem, sa);
  else if (a->la->mode == 2) scan4::scan4_body<2>(a->la->tmap, *a->la->p, a->cta->smem, sa);
  else scan4::scan4_body<0>(a->la->tmap, *a->la->p, a->cta->smem, sa);
  return nullptr;
}

void emu_launch(unsigned grid, const sj_tensor_map &tmap, const ScanParams &p, int mode) {
  const unsigned T = (mode == 3) ? unsigned(utf8v2::kThreadsU) : unsigned(scan4::kThreads4), W = T / 32;
  const size_t smem_bytes = (mode == 3) ? size_t(utf8v2::kSmemBytesU) : size_t(scan4::kSmemBytes4);
  LaunchArgs la{grid, &tmap, &p, mode};
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
      a.la = &la; a.cta = &ctas[c]; a.warp = &warps[c * W + t / 32]; a.tid = t; a.ctaid = c;
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

// what one rank's context and comm hold: scan scratch, the carry slots, and the exchange windows of ALL ranks (in a real
// job each lives on its own GPU; every launch stores its record into each of them)
constexpr size_t kWindowWords = size_t(kXchgSteps) * 2 * kMaxRanks * 2;
struct EmuJob {
  std::vector<unsigned long long> desc;
  uint32_t ticket[4] = {0, 0, 0, 0};
  uint32_t flags = 0;
  uint32_t epoch = 0;
  Carry carry[2];
  std::vector<unsigned long long> window[kMaxRanks];
  EmuJob() { for (auto &w : window) w.assign(kWindowWords, 0ull); }
};

int g_fail = 0;
#define EXPECT(cond, ...)                                       \
  do {                                                          \
    if (!(cond)) {                                              \
      fprintf(stderr, "FAIL %s:%d: %s: ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                             \
      fprintf(stderr, "\n");                                    \
      g_fail++;                                                 \
    }                                                           \
  } while (0)

// One launch over a whole shard, like sharded_enqueue / scan_from_state: kind 0 stage 1, 1 minify, 2 validate_utf8.
// nranks > 0: the last CTA stores the record for (seq, rank) into every window.  Returns the launch's carry out.
Carry launch_shard(EmuJob &J, int kind, const uint8_t *buf, size_t len, uint32_t state_in, uint32_t *idx, uint8_t *dst, unsigned grid,
                   uint32_t nranks, uint32_t rank, uint32_t seq) {
  const uint32_t ntiles = uint32_t((len + kTileBytes - 1) / kTileBytes);
  sj_tensor_map tmap;
  tmap.base = buf; tmap.rows = len / 128; tmap.box_rows = scan4::kBlockRows;
  const bool tma = (reinterpret_cast<uintptr_t>(buf) & 15u) == 0 && tmap.rows > 0;
  ScanParams p;
  memset(&p, 0, sizeof(p));
  p.buf = buf; p.len = len; p.prev_word = 0x20202020u; p.check_eof = 1; p.use_tma = tma ? 1u : 0u;
  p.tile_begin = 0; p.ntiles = ntiles;
  p.flags = &J.flags; p.ticket = J.ticket;
  J.carry[0] = Carry(); J.carry[0].state = state_in & 7u;
  J.carry[1] = Carry();
  p.carry_in = state_in ? &J.carry[0] : nullptr;
  p.carry_out = &J.carry[1];
  for (uint32_t r = 0; r < nranks; r++) p.xchg.peer[r] = J.window[r].data();
  p.xchg.nranks = nranks; p.xchg.rank = rank; p.xchg.slot = (seq % uint32_t(kXchgSteps)) * 2u; p.xchg.seq = seq;
  unsigned g = grid;
  if (kind == kUtf8) {
    emu_launch(g, tmap, p, 3);
    EXPECT(J.ticket[1] == 0 && J.flags == 0, "utf8v2 ticket/flags not re-armed");
    return J.carry[1];
  }
  if (J.desc.size() < size_t(ntiles) + 1) J.desc.assign(size_t(ntiles) + 1, 0ull);
  p.epoch = ++J.epoch;
  p.idx_out = idx; p.dst = dst;
  p.write_sentinels = kind == kIndex ? 1u : 0u;
  p.count_desc = J.desc.data();
  g = std::min<unsigned>(grid, unsigned((uint64_t(ntiles) * kTileBytes + scan4::kElemBytes - 1) / scan4::kElemBytes));
  emu_launch(g, tmap, p, kind == kMinify ? 2 : 0);
  EXPECT(J.ticket[0] == 0 && J.ticket[1] == 0 && J.ticket[2] == 0 && J.flags == 0, "scan4 ticket/flags not re-armed");
  return J.carry[1];
}

// the record (seq, rank) as every window holds it; false when the windows disagree or it is missing
bool read_record(const EmuJob &J, uint32_t nranks, uint32_t rank, uint32_t seq, unsigned long long *w0, unsigned long long *w1) {
  const size_t at = (size_t((seq % uint32_t(kXchgSteps)) * 2u) * kMaxRanks + rank) * 2;
  *w0 = J.window[0][at]; *w1 = J.window[0][at + 1];
  for (uint32_t r = 1; r < nranks; r++)
    if (J.window[r][at] != *w0 || J.window[r][at + 1] != *w1) return false;
  return xchg_complete(*w0, *w1, seq);
}

// minify's kept bytes of buf entered in `state` (bits 0-1), from the oracle: sjo_minify of a document that first reaches
// that state (a quote, a backslash) and, if the shard ends inside a string, closes it -- every added byte is kept
std::vector<uint8_t> oracle_kept(const uint8_t *buf, size_t len, uint32_t state) {
  std::string pre, post;
  if (state & 2u) pre += '"';
  if (state & 1u) pre += '\\';
  uint32_t so = 0;
  std::vector<uint8_t> eq(pre.begin(), pre.end());
  eq.insert(eq.end(), buf, buf + len);
  sjo_scan_shard(eq.data(), eq.size(), 0, nullptr, &so);
  if (so & 1u) post += 'x';
  if (so & 2u) post += '"';
  eq.insert(eq.end(), post.begin(), post.end());
  std::vector<uint8_t> out(eq.size());
  size_t n = 0;
  if (sjo_minify(eq.data(), eq.size(), out.data(), &n) != SJO_SUCCESS || n < pre.size() + post.size()) {
    fprintf(stderr, "oracle_kept: closer failed\n");
    exit(2);
  }
  return std::vector<uint8_t>(out.begin() + long(pre.size()), out.begin() + long(n - post.size()));
}

uint32_t state_after(const uint8_t *buf, size_t len, uint32_t state_in) {
  uint32_t so = 0;
  sjo_scan_shard(buf, len, state_in, nullptr, &so);
  return so & 7u;
}

// ------------------------------------------------------------------ inputs
std::vector<uint8_t> json_rows(std::mt19937_64 &rng, size_t target) {
  const char *words[] = {"a", "\\\\", "\\\"", "\\n", "\xc3\xa9", "\xe2\x82\xac", "\xf0\x9f\x98\x80", "x y", "\\\\\\\"", "q"};
  std::string s;
  while (s.size() < target) {
    s += "{\"id\": " + std::to_string(rng() % 100000) + ",  \"s\" : \"";
    for (int k = int(rng() % 12); k >= 0; k--) s += words[rng() % 10];
    s += "\", \"v\":\t[1, 2 ,\n  true, \"";
    for (int k = int(rng() % 6); k >= 0; k--) s += words[rng() % 10];
    s += "\"]}\n";
    if (rng() % 5 == 0) s += std::string(rng() % 300, ' ');
  }
  return std::vector<uint8_t>(s.begin(), s.end());
}

std::vector<uint8_t> backslash_runs(std::mt19937_64 &rng, size_t target) {
  std::string s = "[";
  while (s.size() < target) {
    s += " \"";
    const size_t run = rng() % 2 ? rng() % 40 : 4095 + rng() % 3;
    s += std::string(run + (run & 1), '\\');  // even runs: the closing quote is not escaped
    s += "\" ,";
  }
  s += "0]";
  return std::vector<uint8_t>(s.begin(), s.end());
}

std::vector<uint8_t> utf8_text(std::mt19937_64 &rng, size_t target) {
  const char *cps[] = {"a", " ", "\xc3\xa9", "\xe2\x82\xac", "\xf0\x9f\x98\x80", "\xdf\xbf", "Z"};
  std::string s;
  while (s.size() < target) s += cps[rng() % 7];
  return std::vector<uint8_t>(s.begin(), s.end());
}

// cuts at arbitrary bytes, with some placed just after a backslash and some inside a string
std::vector<size_t> minify_cuts(std::mt19937_64 &rng, const std::vector<uint8_t> &doc, int nranks) {
  std::vector<size_t> cuts{0};
  for (int k = 1; k < nranks; k++) {
    size_t c = doc.size() * size_t(k) / size_t(nranks) + rng() % 97;
    const int how = int(rng() % 3);
    for (size_t i = c; i < doc.size() - 1 && i < c + 4000; i++) {
      if (how == 0 && doc[i - 1] == '\\') { c = i; break; }                                  // just after a backslash
      if (how == 1 && (state_after(doc.data(), i, 0) & 2u)) { c = i; break; }                // inside a string
    }
    cuts.push_back(std::max(cuts.back() + 1, std::min(c, doc.size() - 1)));
  }
  cuts.push_back(doc.size());
  return cuts;
}

// ------------------------------------------------------------------ checks
// every rank's speculative minify launch (state 0) publishes its record; ranks whose true incoming state has bit 0 or 1
// set minify again from that state (the second round); the kept bytes at the ranks' bases are the whole buffer's minify
int check_minify(EmuJob &J, std::mt19937_64 &rng, const std::vector<uint8_t> &doc, const std::vector<size_t> &cuts, uint32_t seq, const char *what) {
  const uint32_t nranks = uint32_t(cuts.size() - 1);
  std::vector<uint8_t> whole(doc.size());
  size_t wlen = 0;
  const bool closed = sjo_minify(doc.data(), doc.size(), whole.data(), &wlen) == SJO_SUCCESS;
  const std::vector<uint8_t> want = closed ? std::vector<uint8_t>(whole.begin(), whole.begin() + long(wlen)) : oracle_kept(doc.data(), doc.size(), 0);
  size_t base = 0;
  int rescans = 0;
  for (uint32_t r = 0; r < nranks; r++) {
    const uint8_t *buf = doc.data() + cuts[r];
    const size_t len = cuts[r + 1] - cuts[r];
    std::vector<uint8_t> store(len + 16);
    uint8_t *sb = store.data() + ((rng() % 4 == 0) ? 1 + rng() % 15 : 0);  // misaligned shards: plain loads
    if (sb + len > store.data() + store.size()) sb = store.data();
    memcpy(sb, buf, len);
    std::vector<uint8_t> dst(len + 64, 0xEE);
    const unsigned grid = 1 + unsigned(rng() % 3);
    const Carry spec = launch_shard(J, kMinify, sb, len, 0, nullptr, dst.data(), grid, nranks, r, seq);
    unsigned long long w0 = 0, w1 = 0;
    const std::vector<uint8_t> k0 = oracle_kept(sb, len, 0);
    EXPECT(read_record(J, nranks, r, seq, &w0, &w1), "%s rank %u: record missing", what, r);
    EXPECT(xchg_kind(w1) == kMinify && xchg_count(w0) == k0.size() && spec.count == k0.size(), "%s rank %u: kind %d count %llu want %zu", what, r,
           xchg_kind(w1), (unsigned long long)xchg_count(w0), k0.size());
    EXPECT((w1 & 7u) == state_after(sb, len, 0) && ((w1 >> 8) & 0x3Fu) == sjo_transducer(sb, len) && ((w1 >> 16) & 0xFFu) == 0,
           "%s rank %u: state %llu tt %llu flags %llu want state %u tt %u", what, r, w1 & 7u, (w1 >> 8) & 0x3Fu, (w1 >> 16) & 0xFFu,
           state_after(sb, len, 0), sjo_transducer(sb, len));
    const uint32_t s_true = state_after(doc.data(), cuts[r], 0);
    std::vector<uint8_t> got(dst.begin(), dst.begin() + long(spec.count));
    if (s_true & 3u) {
      std::fill(dst.begin(), dst.end(), 0xEE);
      const Carry again = launch_shard(J, kMinify, sb, len, s_true, nullptr, dst.data(), grid, 0, 0, 0);
      got.assign(dst.begin(), dst.begin() + long(again.count));
      EXPECT(again.state == state_after(sb, len, s_true), "%s rank %u: state after re-minify %u", what, r, again.state);
      for (size_t i = size_t(again.count); i < dst.size(); i++)
        if (dst[i] != 0xEE) { EXPECT(false, "%s rank %u: wrote past the kept bytes at %zu", what, r, i); break; }
      rescans++;
    }
    const bool same = base + got.size() <= want.size() && memcmp(got.data(), want.data() + base, got.size()) == 0;
    EXPECT(same, "%s rank %u of %u: kept bytes differ from the whole buffer's minify at base %zu (count %zu, state_in %u, cut %zu)", what, r, nranks,
           base, got.size(), s_true, cuts[r]);
    base += got.size();
  }
  EXPECT(base == want.size(), "%s: total %zu want %zu", what, base, want.size());
  return rescans;
}

// stage-1 records keep kind 0 and their previous layout
void check_stage1_record(EmuJob &J, const std::vector<uint8_t> &shard, uint32_t seq) {
  std::vector<uint32_t> idx(shard.size() + 16);
  const Carry c = launch_shard(J, kIndex, shard.data(), shard.size(), 0, idx.data(), nullptr, 2, 3, 1, seq);
  unsigned long long w0 = 0, w1 = 0;
  uint32_t so = 0;
  const uint64_t n = sjo_scan_shard(shard.data(), shard.size(), 0, nullptr, &so);
  const uint32_t fl = sjo_validate_utf8(shard.data(), shard.size()) ? 0u : uint32_t(kFlagUtf8);
  EXPECT(read_record(J, 3, 1, seq, &w0, &w1), "stage-1 record missing");
  EXPECT(w0 == xchg_word0(seq, n) && w1 == xchg_word1(seq, so & 7u, sjo_transducer(shard.data(), shard.size()), c.flags, kIndex) && c.count == n &&
             (c.flags & ~uint32_t(kFlagCtl)) == fl,
         "stage-1 record w0 %llx w1 %llx n %llu flags %u", w0, w1, (unsigned long long)n, c.flags);
  EXPECT(xchg_kind(w1) == kIndex && (w1 >> 24 & 0xFFu) == 0, "stage-1 record kind bits %llx", w1);
}

// utf8v2: every shard (cut at character boundaries) publishes {0, 0, 0, flags, kind 2}; the OR of the flags is the verdict
void check_utf8(EmuJob &J, std::mt19937_64 &rng, std::vector<uint8_t> text, int nranks, int corrupt_rank, int corrupt_where, uint32_t seq) {
  std::vector<size_t> cuts{0};
  for (int k = 1; k < nranks; k++) {
    size_t c = text.size() * size_t(k) / size_t(nranks) + rng() % 50;
    for (int j = 0; j < 3 && (text[c] & 0xC0) == 0x80; j++) c--;  // sjb200_shard_cut
    cuts.push_back(c);
  }
  cuts.push_back(text.size());
  if (corrupt_rank >= 0) {
    const size_t lo = cuts[size_t(corrupt_rank)], hi = cuts[size_t(corrupt_rank) + 1];
    const size_t at = corrupt_where == 0 ? lo : corrupt_where == 1 ? (lo + hi) / 2 : hi - 1 - rng() % 3;
    text[at] = uint8_t(corrupt_where == 2 ? 0xE2 : 0xFF);  // (at the end: a lead byte whose sequence is cut short)
  }
  uint32_t any = 0;
  for (int r = 0; r < nranks; r++) {
    const uint8_t *buf = text.data() + cuts[size_t(r)];
    const size_t len = cuts[size_t(r) + 1] - cuts[size_t(r)];
    const Carry c = launch_shard(J, kUtf8, buf, len, 0, nullptr, nullptr, 1 + unsigned(rng() % 3), uint32_t(nranks), uint32_t(r), seq);
    unsigned long long w0 = 0, w1 = 0;
    const bool valid = sjo_validate_utf8(buf, len) != 0;
    EXPECT(read_record(J, uint32_t(nranks), uint32_t(r), seq, &w0, &w1), "utf8 rank %d: record missing", r);
    EXPECT(w0 == xchg_word0(seq, 0) && w1 == xchg_word1(seq, 0, 0, valid ? 0u : uint32_t(kFlagUtf8), kUtf8) && c.flags == (valid ? 0u : uint32_t(kFlagUtf8)),
           "utf8 rank %d of %d (corrupt rank %d where %d): w0 %llx w1 %llx valid %d", r, nranks, corrupt_rank, corrupt_where, w0, w1, int(valid));
    any |= uint32_t(w1 >> 16) & 0xFFu;
  }
  const bool whole = sjo_validate_utf8(text.data(), text.size()) != 0;
  EXPECT(whole == !(any & kFlagUtf8), "utf8: AND of the shard verdicts %d, whole buffer %d", int(!(any & kFlagUtf8)), int(whole));
  EXPECT(whole == (corrupt_rank < 0), "utf8: the corruption did not make the buffer invalid");
}

}  // namespace

int main(int argc, char **argv) {
  const int iters = argc > 1 ? atoi(argv[1]) : 6;
  std::mt19937_64 rng(0x5A4D5);
  EmuJob J;
  uint32_t seq = 0;
  int rescans = 0;
  // fixed cases first: a cut right after a backslash inside a string, a cut between the two bytes of an escape pair, a
  // buffer that ends inside a string
  {
    std::string s = "{\"k\": \"ab\\\"cd\\\\\", \"t\": [1, 2]}\n";
    while (s.size() < 70000) s += "{\"k\": \"ab\\\"cd\\\\\", \"t\": [1,   2]}\n";
    std::vector<uint8_t> doc(s.begin(), s.end());
    const size_t bs = s.find('\\', 40000);
    rescans += check_minify(J, rng, doc, {0, bs + 1, doc.size()}, ++seq, "after a backslash");
    rescans += check_minify(J, rng, doc, {0, 9, bs, bs + 2, doc.size()}, ++seq, "inside strings");
    std::vector<uint8_t> open = doc;
    open.push_back('"');
    for (int i = 0; i < 5000; i++) open.push_back("ab \\\n"[i % 4]);
    rescans += check_minify(J, rng, open, {0, 30000, 69000, open.size()}, ++seq, "ends inside a string");
  }
  for (int it = 0; it < iters && g_fail < 5; it++) {
    const int nranks = 2 + int(rng() % 7);
    const std::vector<uint8_t> doc = (it % 2 == 0) ? json_rows(rng, 20000 + rng() % 180000) : backslash_runs(rng, 20000 + rng() % 100000);
    rescans += check_minify(J, rng, doc, minify_cuts(rng, doc, nranks), ++seq, it % 2 == 0 ? "rows" : "backslash runs");
  }
  check_stage1_record(J, json_rows(rng, 90000), ++seq);
  const std::vector<uint8_t> text = utf8_text(rng, 150000);
  check_utf8(J, rng, text, 4, -1, 0, ++seq);
  for (int where = 0; where < 3; where++) check_utf8(J, rng, text, 3, int(rng() % 3), where, ++seq);
  check_utf8(J, rng, text, 2, 1, 2, ++seq);  // the last bytes of the document
  EXPECT(rescans >= 4, "only %d shards started with escape / in-string set", rescans);
  if (g_fail) { printf("FAILED\n"); return 1; }
  printf("simt emulation of sharded minify / validate_utf8 records OK (%d cases, %d shards minified again from their true state)\n", iters, rescans);
  return 0;
}
