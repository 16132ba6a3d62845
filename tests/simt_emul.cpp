// simt_emul.cpp -- runs the ACTUAL scan4 kernel source (simdjson_b200/csrc/sjb200_scan4.cuh) on the CPU and checks it
// against the oracle.
//
// The kernel is written against the small primitive set of sjb200_simt.cuh; with SJB200_HOST_EMU those primitives are
// implemented with one OS thread per CUDA thread (warp collectives = 32-thread rendezvous, mbarriers with deferred TMA
// copies, atomics on plain memory).  Everything else -- warp roles, the ticket / mbarrier pipeline, both-polarity block
// scans, the decoupled look-back chain, emit, launch finalisation -- is the code the GPU runs.  This catches protocol and
// algebra bugs on a machine without a GPU; it does not model the GPU memory model or timing.  Test infrastructure only.
//
// build: see tests/test_simt_emul.py
#define SJB200_HOST_EMU 1
#include "sjb200_scan4.cuh"
#include "sjb200_utf8.cuh"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <thread>
#include <vector>

#include "simt_fenced.h"

extern "C" {
#include "sj_oracle.h"
}

using namespace sjb200;

thread_local simt::ThreadCtx simt::tctx;

namespace {

struct LaunchArgs {
  unsigned grid;
  const sj_tensor_map *tmap;
  const ScanParams *p;
  int mode;  // 0 stage 1, 2 minify, 3 validate_utf8 (utf8v2)
};

void *thread_main(void *arg);
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


// what the context keeps (sjb200_ctx.h)
struct EmuCtx {
  std::vector<unsigned long long> desc;
  uint32_t ticket[4] = {0, 0, 0, 0};
  uint32_t flags = 0;
  uint32_t epoch = 0;
  Carry carry[64];
};

struct Result {
  uint64_t count = 0;
  uint32_t state = 0, ttable = 0, flags = 0;
  std::vector<uint32_t> idx;
};

// one document (or shard) through 1..n launches of chunk_tiles tiles each, like scan_host_document
// (idx_ext: the index output goes there instead of into Result::idx)
Result run_scan4(EmuCtx &cx, const uint8_t *buf, size_t len, uint32_t state_in, uint32_t chunk_tiles, unsigned grid, bool use_tma,
                 bool sentinels, uint8_t *minify_dst = nullptr, uint32_t *idx_ext = nullptr) {
  Result r;
  const uint32_t ntiles_total = uint32_t((len + kTileBytes - 1) / kTileBytes);
  if (cx.desc.size() < size_t(ntiles_total) + 1) cx.desc.assign(size_t(ntiles_total) + 1, 0ull);
  if (!idx_ext) r.idx.assign(len + 80, 0xABABABABu);
  sj_tensor_map tmap;
  tmap.base = buf;
  tmap.rows = len / 128;
  tmap.box_rows = scan4::kBlockRows;
  const bool tma_ok = use_tma && (reinterpret_cast<uintptr_t>(buf) & 15u) == 0 && tmap.rows > 0;
  if (chunk_tiles == 0) chunk_tiles = ntiles_total;
  cx.carry[0].count = 0; cx.carry[0].state = state_in & 7u; cx.carry[0].ttable = 0; cx.carry[0].flags = 0; cx.carry[0].reserved = 0;
  int slot = 0;
  uint32_t flags = 0;
  for (uint32_t tb = 0; tb < ntiles_total; tb += chunk_tiles) {
    const uint32_t nt = std::min(chunk_tiles, ntiles_total - tb);
    ScanParams p;
    memset(&p, 0, sizeof(p));
    p.buf = buf; p.len = len; p.pos_base = 0; p.prev_word = 0x20202020u;
    p.check_eof = (tb + nt == ntiles_total) ? 1u : 0u;
    p.use_tma = tma_ok ? 1u : 0u;
    p.tile_begin = tb; p.ntiles = nt;
    p.epoch = ++cx.epoch;
    p.idx_out = idx_ext ? idx_ext : r.idx.data(); p.dst = minify_dst;
    p.write_sentinels = (sentinels && !minify_dst && tb + nt == ntiles_total) ? 1u : 0u;
    p.carry_in = &cx.carry[slot];
    p.carry_out = &cx.carry[slot + 1];
    p.flags = &cx.flags; p.count_desc = cx.desc.data(); p.ticket = cx.ticket; p.debug = nullptr;
    cx.carry[slot + 1] = Carry();
    const unsigned g = std::min<unsigned>(grid, (nt * unsigned(kTileBytes) + scan4::kElemBytes - 1) / scan4::kElemBytes);
    emu_launch(g, tmap, p, minify_dst ? 2 : 0);
    if (cx.ticket[0] != 0 || cx.ticket[1] != 0 || cx.ticket[2] != 0 || cx.flags != 0) { fprintf(stderr, "BUG: ticket/flags not re-armed\n"); exit(2); }
    flags |= cx.carry[slot + 1].flags;
    slot++;
    if (slot + 1 >= 64) { fprintf(stderr, "too many chunks\n"); exit(2); }
  }
  r.count = cx.carry[slot].count;
  r.state = cx.carry[slot].state;
  r.ttable = cx.carry[slot].ttable;
  r.flags = flags;
  return r;
}

int g_fail = 0;

void hexdump(const std::vector<uint8_t> &in) {
  fprintf(stderr, "  hex:");
  for (size_t i = 0; i < in.size() && i < 300; i++) fprintf(stderr, "%02x", in[i]);
  fprintf(stderr, "\n");
}

int check(EmuCtx &cx, const std::vector<uint8_t> &store, size_t misalign, uint32_t state_in, uint32_t chunk_tiles, unsigned grid, bool use_tma,
          const char *what) {
  const uint8_t *buf = store.data() + misalign;
  const size_t len = store.size() - misalign;
  if (len == 0) return 0;
  Result r = run_scan4(cx, buf, len, state_in, chunk_tiles, grid, use_tma, true);
  std::vector<uint32_t> oidx(len + 16);
  uint32_t ostate = 0;
  const uint64_t on = sjo_scan_shard(buf, len, state_in, oidx.data(), &ostate);
  int bad = 0;
  if (r.flags & kFlagInternal) bad = 1;
  else if (r.count != on) bad = 2;
  else if (memcmp(r.idx.data(), oidx.data(), on * 4) != 0) bad = 3;
  else if (r.idx[on] != uint32_t(len) || r.idx[on + 1] != uint32_t(len) || r.idx[on + 2] != 0) bad = 4;
  else if (r.state != (ostate & 7u)) bad = 5;
  else if (bool(r.flags & kFlagUtf8) == bool(sjo_validate_utf8(buf, len))) bad = 6;
  if (!bad && chunk_tiles == 0) {
    const uint32_t ott = sjo_transducer(buf, len);
    if (r.ttable != ott) bad = 7;
  }
  if (!bad) {
    // unescaped control character inside a string: ask the oracle about an equivalent document that starts in state 0
    std::vector<uint8_t> eq;
    if (state_in & 2u) eq.push_back('"');
    if (state_in & 1u) eq.push_back('\\');
    eq.insert(eq.end(), buf, buf + len);
    std::vector<uint32_t> tmp(sjo_index_capacity(eq.size()) + 16);
    uint32_t n = 0;
    // (streaming_final tolerates an unclosed string, so UNESCAPED_CHARS is reported whenever the flag is due)
    size_t elen = eq.size();
    while (elen > 0 && (eq[elen - 1] & 0x80u)) elen--;  // keep clear of the partial-UTF-8 trimming of streaming modes
    if (elen > 0) {
      const int oerr = sjo_stage1(eq.data(), elen, elen, SJO_STREAMING_FINAL, tmp.data(), &n);
      if (elen == eq.size() && bool(r.flags & kFlagCtl) != (oerr == SJO_UNESCAPED_CHARS)) bad = 8;
    }
  }
  if (bad) {
    fprintf(stderr, "MISMATCH kind=%d (%s) len=%zu misalign=%zu state_in=%u chunk_tiles=%u grid=%u tma=%d: got n=%llu state=%u tt=%u flags=%u | want n=%llu state=%u\n",
            bad, what, len, misalign, state_in, chunk_tiles, grid, int(use_tma), (unsigned long long)r.count, r.state, r.ttable, r.flags,
            (unsigned long long)on, ostate);
    if (bad == 3)
      for (uint64_t i = 0; i < on; i++)
        if (r.idx[i] != oidx[i]) { fprintf(stderr, "  first difference at output %llu: got %u want %u\n", (unsigned long long)i, r.idx[i], oidx[i]); break; }
    std::vector<uint8_t> v(buf, buf + len);
    hexdump(v);
    g_fail++;
  }
  return bad;
}

// ---- the look-back fold on its own: one emulated warp against a scalar walk, with the nearest inclusive prefix up to
// three windows away and stale / missing descriptors behind it (the multi-CTA runs above only reach short distances)
struct LbArgs {
  const ScanParams *p;
  uint32_t t;
  simt::WarpShared *warp;
  simt::CtaShared *cta;
  unsigned lane;
  uint32_t s_in, base;
};
void *lb_thread(void *arg) {
  LbArgs *a = static_cast<LbArgs *>(arg);
  simt::tctx = simt::ThreadCtx();
  simt::tctx.tid = a->lane;
  simt::tctx.nctas = 1;
  simt::tctx.warp = a->warp;
  simt::tctx.ctas = a->cta;
  scan4::look_back(*a->p, a->t, a->lane, &a->s_in, &a->base);
  return nullptr;
}
int test_look_back(std::mt19937_64 &rng, int cases) {
  int bad = 0;
  for (int c = 0; c < cases && bad < 3; c++) {
    const uint32_t t = 1 + uint32_t(rng() % 1500);
    const uint32_t epoch = 1 + uint32_t(rng() % 1000);
    std::vector<unsigned long long> desc(t + 1, 0ull);
    uint32_t flags = 0;
    // nearest inclusive prefix at `inc`; everything newer is an aggregate; older entries are junk that must not matter
    const uint32_t maxback = std::min<uint32_t>(t, 1 + uint32_t(rng() % 1000));
    const uint32_t inc = t - 1 - uint32_t(rng() % maxback);
    const uint32_t s_k = uint32_t(rng() & 1), c_k = uint32_t(rng() % 100000000u);
    for (uint32_t i = 0; i < t; i++) {
      const uint32_t par = uint32_t(rng() & 1), c0 = uint32_t(rng() % 32769), c1 = uint32_t(rng() % 32769);
      if (i > inc) desc[i] = scan4::pack_agg(epoch, par, c0, c1);
      else if (i == inc) desc[i] = scan4::pack_inc(epoch, s_k, c_k);
      else {
        const int kind = int(rng() % 4);
        desc[i] = kind == 0 ? 0ull : kind == 1 ? scan4::pack_agg(epoch - 1, par, c0, c1) : kind == 2 ? scan4::pack_inc(epoch, par, c0) : scan4::pack_agg(epoch, par, c0, c1);
      }
    }
    desc[0] = (inc == 0) ? desc[0] : scan4::pack_inc(epoch, uint32_t(rng() & 1), 12345);  // element 0 is always inclusive
    uint32_t s = s_k;
    uint64_t cnt = c_k;
    for (uint32_t i = inc + 1; i < t; i++) {
      const unsigned long long d = desc[i];
      cnt += s ? (uint32_t(d >> 19) & 0x7FFFFu) : (uint32_t(d) & 0x7FFFFu);
      s ^= uint32_t(d >> 38) & 1u;
    }
    ScanParams p;
    memset(&p, 0, sizeof(p));
    p.epoch = epoch; p.count_desc = desc.data(); p.flags = &flags;
    simt::WarpShared w;
    simt::CtaShared cta;
    pthread_barrier_init(&w.bar, nullptr, 32);
    std::vector<LbArgs> args(32);
    std::vector<pthread_t> th(32);
    for (unsigned l = 0; l < 32; l++) {
      args[l] = LbArgs{&p, t, &w, &cta, l, 0, 0};
      pthread_create(&th[l], nullptr, lb_thread, &args[l]);
    }
    for (auto &x : th) pthread_join(x, nullptr);
    pthread_barrier_destroy(&w.bar);
    for (unsigned l = 0; l < 32; l++)
      if (args[l].s_in != s || args[l].base != uint32_t(cnt) || flags != 0) {
        fprintf(stderr, "LOOK-BACK MISMATCH t=%u inc=%u lane=%u: got (%u,%u) want (%u,%u) flags=%u\n", t, inc, l, args[l].s_in, args[l].base, s, uint32_t(cnt), flags);
        bad++;
        break;
      }
  }
  return bad;
}

// minify on the scan4 structure against the oracle (json_minifier.h semantics: bytes and length when the document has no
// unclosed string; UNCLOSED_STRING otherwise; nothing is ever written past dst[len))
int check_minify(EmuCtx &cx, const std::vector<uint8_t> &store, size_t misalign, uint32_t chunk_tiles, unsigned grid, bool use_tma, size_t dst_misalign) {
  const uint8_t *buf = store.data() + misalign;
  const size_t len = store.size() - misalign;
  if (len == 0) return 0;
  std::vector<uint8_t> out(len + 64 + dst_misalign, 0xEE);
  uint8_t *dst = out.data() + dst_misalign;
  Result r = run_scan4(cx, buf, len, 0, chunk_tiles, grid, use_tma, false, dst);
  std::vector<uint8_t> want(len + 1);
  size_t wlen = 0;
  const int werr = sjo_minify(buf, len, want.data(), &wlen);
  int bad = 0;
  const bool unclosed = (r.state >> 1) & 1u;
  if (r.flags & kFlagInternal) bad = 1;
  else if (unclosed != (werr == SJO_UNCLOSED_STRING)) bad = 2;
  else if (!unclosed && (r.count != wlen || memcmp(dst, want.data(), wlen) != 0)) bad = 3;
  else {
    for (size_t i = size_t(r.count); i < len + 64 && !bad; i++)
      if (dst[i] != 0xEE) bad = 4;  // wrote beyond the kept bytes
    for (size_t i = 0; i < dst_misalign && !bad; i++)
      if (out[i] != 0xEE) bad = 5;
  }
  if (bad) {
    fprintf(stderr, "MINIFY MISMATCH kind=%d len=%zu misalign=%zu dst_misalign=%zu chunk_tiles=%u grid=%u tma=%d: got n=%llu | want err=%d n=%zu\n", bad, len, misalign,
            dst_misalign, chunk_tiles, grid, int(use_tma), (unsigned long long)r.count, werr, wlen);
    if (bad == 3)
      for (size_t i = 0; i < wlen; i++)
        if (dst[i] != want[i]) { fprintf(stderr, "  first difference at output byte %zu: got %02x want %02x\n", i, dst[i], want[i]); break; }
    std::vector<uint8_t> v(buf, buf + len);
    hexdump(v);
    g_fail++;
  }
  return bad;
}

// validate_utf8 with independent warps (sjb200_utf8.cuh) against the oracle; chunk_tiles > 0: several launches like the host path
int check_utf8v2(EmuCtx &cx, const uint8_t *buf, size_t len, size_t misalign, uint32_t chunk_tiles, unsigned grid, bool use_tma) {
  if (len == 0) return 0;
  const uint32_t ntiles_total = uint32_t((len + kTileBytes - 1) / kTileBytes);
  sj_tensor_map tmap;
  tmap.base = buf; tmap.rows = len / 128; tmap.box_rows = utf8v2::kBlockRowsU;
  const bool tma_ok = use_tma && (reinterpret_cast<uintptr_t>(buf) & 15u) == 0 && tmap.rows > 0;
  if (chunk_tiles == 0) chunk_tiles = ntiles_total;
  uint32_t flags = 0;
  for (uint32_t tb = 0; tb < ntiles_total; tb += chunk_tiles) {
    const uint32_t nt = std::min(chunk_tiles, ntiles_total - tb);
    ScanParams p;
    memset(&p, 0, sizeof(p));
    p.buf = buf; p.len = len; p.prev_word = 0x20202020u;
    p.check_eof = (tb + nt == ntiles_total) ? 1u : 0u;
    p.use_tma = tma_ok ? 1u : 0u;
    p.tile_begin = tb; p.ntiles = nt;
    p.carry_out = &cx.carry[1];
    p.flags = &cx.flags; p.ticket = cx.ticket;
    cx.carry[1] = Carry();
    emu_launch(grid, tmap, p, 3);
    if (cx.ticket[1] != 0 || cx.flags != 0) { fprintf(stderr, "BUG: utf8v2 ticket/flags not re-armed\n"); exit(2); }
    flags |= cx.carry[1].flags;
  }
  const bool got = !(flags & kFlagUtf8), want = sjo_validate_utf8(buf, len) != 0;
  if (got != want || (flags & kFlagInternal)) {
    fprintf(stderr, "UTF8V2 MISMATCH len=%zu misalign=%zu chunk_tiles=%u grid=%u tma=%d: got %d want %d flags=%u\n", len, misalign, chunk_tiles, grid, int(use_tma), int(got), int(want), flags);
    std::vector<uint8_t> v(buf, buf + len);
    hexdump(v);
    g_fail++;
    return 1;
  }
  return 0;
}
int check_utf8v2(EmuCtx &cx, const std::vector<uint8_t> &store, size_t misalign, uint32_t chunk_tiles, unsigned grid, bool use_tma) {
  return check_utf8v2(cx, store.data() + misalign, store.size() - misalign, misalign, chunk_tiles, grid, use_tma);
}

// ---- fenced pass: every buffer the kernels are given is exactly as long as the C API promises and sits right against a
// PROT_NONE page, so a read of the input or a write of an output outside its bounds kills the process instead of going
// unnoticed (the TMA full-block predicate, the guarded fill of the last block, the look-backs before byte 0, the 16-byte
// copy-outs of the stage-1 and minify emits, the sentinel words)
// (Fenced, index_words: simt_fenced.h)

// a document that changes its result if one byte more is read at either end: it starts with a continuation byte, a quote,
// a backslash or a digit and ends in a backslash, an open string, a partial or complete UTF-8 character, a number or a
// truncated atom; backslash runs and quotes sit on the block boundaries in between
std::vector<uint8_t> fenced_doc(std::mt19937_64 &rng, size_t len) {
  static const char *alpha = "\\\\\\\"\" {}[],: \n\tabc1\x01\x1e";
  static const char *heads[] = {"\x80", "\"", "\\", "7"};
  static const char *tails[] = {"\\", "\"ab", "\xf0\x9f\x98", "\xe2\x82\xac", "123", "tru", "\xc3"};
  std::vector<uint8_t> d(len);
  const size_t alen = strlen(alpha);
  for (size_t i = 0; i < len; i++) d[i] = uint8_t(rng() % 3 ? alpha[rng() % alen] : 'a' + rng() % 26);
  for (size_t b = 128; b + 8 < len; b += 128)
    if (b % 4096 == 0 || rng() % 8 == 0) {
      const size_t run = 1 + rng() % 5;
      for (size_t k = 0; k < run && b - k > 0; k++) d[b - k] = '\\';
      if (rng() % 2) d[b + 1] = '"';
    }
  if (len == 0) return d;
  const char *h = heads[rng() % 4];
  d[0] = uint8_t(h[0]);
  const char *t = tails[rng() % 7];
  const size_t tl = std::min(strlen(t), len);
  memcpy(d.data() + len - tl, t + strlen(t) - tl, tl);
  return d;
}

int fenced_case(EmuCtx &cx, const std::vector<uint8_t> &doc, bool in_at_end, bool out_at_end, bool use_tma, uint32_t state_in, bool sentinels, unsigned grid,
                bool minify, bool utf8) {
  const size_t len = doc.size();
  Fenced in(len, in_at_end);
  memcpy(in.p, doc.data(), len);
  const uint8_t *buf = in.p;
  int bad = 0;
  {  // stage 1 (sentinels) / a shard that is not the last (sjb200_stage1_shard_dev: none): exactly sjb200_index_words(len) words
    const size_t words = index_words(len);
    Fenced out(words * 4, out_at_end);
    uint32_t *idx = reinterpret_cast<uint32_t *>(out.p);
    for (size_t i = 0; i < words; i++) idx[i] = 0xABABABABu;
    Result r = run_scan4(cx, buf, len, state_in, 0, grid, use_tma, sentinels, nullptr, idx);
    std::vector<uint32_t> oidx(len + 16);
    uint32_t ostate = 0;
    const uint64_t on = sjo_scan_shard(buf, len, state_in, oidx.data(), &ostate);
    if (r.flags & kFlagInternal) bad = 1;
    else if (r.count != on || memcmp(idx, oidx.data(), on * 4) != 0) bad = 2;
    else if (sentinels && (idx[on] != uint32_t(len) || idx[on + 1] != uint32_t(len) || idx[on + 2] != 0)) bad = 3;
    else if (r.state != (ostate & 7u) || r.ttable != sjo_transducer(buf, len)) bad = 4;
    else if (bool(r.flags & kFlagUtf8) == bool(sjo_validate_utf8(buf, len))) bad = 5;
    for (size_t i = on + (sentinels ? 3 : 0); i < words && !bad; i++)
      if (idx[i] != 0xABABABABu) bad = 6;  // a word past the structurals (and sentinels)
  }
  if (!bad && minify) {  // minify: dst exactly len bytes
    Fenced out(len, out_at_end);
    memset(out.p, 0xEE, len);
    Result r = run_scan4(cx, buf, len, 0, 0, grid, use_tma, false, out.p);
    std::vector<uint8_t> want(len + 1);
    size_t wlen = 0;
    const int werr = sjo_minify(buf, len, want.data(), &wlen);
    const bool unclosed = (r.state >> 1) & 1u;
    if (r.flags & kFlagInternal) bad = 11;
    else if (unclosed != (werr == SJO_UNCLOSED_STRING)) bad = 12;
    else if (!unclosed && (r.count != wlen || memcmp(out.p, want.data(), wlen) != 0)) bad = 13;
    for (size_t i = size_t(r.count); i < len && !bad; i++)
      if (out.p[i] != 0xEE) bad = 14;
  }
  if (bad) {
    fprintf(stderr, "FENCED MISMATCH kind=%d len=%zu in_at_end=%d out_at_end=%d tma=%d state_in=%u sentinels=%d grid=%u\n", bad, len, int(in_at_end),
            int(out_at_end), int(use_tma), state_in, int(sentinels), grid);
    hexdump(doc);
    g_fail++;
  }
  if (!bad && utf8) bad = check_utf8v2(cx, buf, len, 0, 0, grid, use_tma);
  return bad;
}

int run_fenced(std::mt19937_64 &rng) {
  EmuCtx cx;
  const size_t T = kTileBytes;
  const size_t lens[] = {1, 3, 4, 5, 16, 127, 128, 129, 4095, 4096, 4097, 8192 + 127, 8192 + 128, T - 1, T, T + 1, 2 * T + 128, 3 * T + 4095};
  int cases = 0;
  for (size_t len : lens) {
    for (int placement = 0; placement < 4; placement++) {
      const bool in_at_end = (placement & 1) == 0, out_at_end = (placement & 2) == 0;
      for (int tma = 1; tma >= 0; tma--) {
        const std::vector<uint8_t> doc = fenced_doc(rng, len);
        const unsigned grid = 1 + unsigned(rng() % 2);
        // every incoming shard state on the short documents, one random state on the long ones
        const uint32_t nstates = len <= 4097 && placement == 0 ? 8u : 1u;
        for (uint32_t s = 0; s < nstates; s++) {
          const uint32_t state_in = nstates == 8 ? s : uint32_t(rng() % 8);
          fenced_case(cx, doc, in_at_end, out_at_end, tma != 0, state_in, (cases & 1) == 0, grid, s == 0, s == 0);
          cases++;
          if (g_fail >= 5) return g_fail;
        }
      }
    }
  }
  printf("fenced pass: %d cases\n", cases);
  return g_fail;
}

}  // namespace

int main(int argc, char **argv) {
  if (argc > 1 && strcmp(argv[1], "--fenced") == 0) {
    std::mt19937_64 frng(0xfe9ced);
    if (run_fenced(frng)) { printf("FAILED\n"); return 1; }
    printf("simt emulation, fenced buffers OK\n");
    return 0;
  }
  const int iters = argc > 1 ? atoi(argv[1]) : 120;
  std::mt19937_64 rng(0x5eed1234);
  const char *alphabets[] = {"\\\\\\\"\" {}[],: \n\tabc1\x01\x0c\x1a\x1e", "\\\"", "\\\\\\\\\\\\\\\"a ", "\"{}[],:0 ", " \n\r\t\"a\\", ",{}[] 1 \"a\":\n"};
  const char *utf8bits[] = {"\xc3\xa9", "\xe2\x82\xac", "\xf0\x9f\x98\x80", "\xff", "\xc3", "\xe2\x82", "\xf0\x9f\x98", "\x80", "\xed\xa0\x80", "\xc0\xaf", "\xf4\x90\x80\x80", "\xe0\x9f\xbf", "\xf0\x8f\xbf\xbf", "\xf5\x80\x80\x80", "\xed\x9f\xbf", "\xf4\x8f\xbf\xbf", "\xe0\xa0\x80", "\xf0\x90\x80\x80", "\xc2\x80", "\xdf\xbf"};
  EmuCtx cx;
  g_fail += test_look_back(rng, 300);
  for (int it = 0; it < iters && g_fail < 5; it++) {
    std::vector<uint8_t> in;
    const int kind = int(rng() % 8);
    uint32_t force_state = 0xFFFFFFFFu;
    const char *a = alphabets[rng() % 6];
    const size_t alen = strlen(a);
    size_t n = rng() % 3000;
    if (kind == 0) {  // long backslash runs around lane / block / element boundaries
      size_t pre = rng() % 3 ? (rng() % 5) * 128 + (rng() % 9) + 4096 * (rng() % 9) : rng() % 300;
      if (pre >= 4) pre -= rng() % 5;
      for (size_t i = 0; i < pre; i++) in.push_back(uint8_t(a[rng() % alen]));
      const size_t runs[] = {1, 2, 3, 15, 16, 17, 31, 32, 33, 127, 128, 129, 4095, 4096, 4097, 8191, 8192, 8193};
      const size_t run = ((rng() % 10 == 0) ? size_t(33000) : runs[rng() % 18]) + rng() % 2;
      for (size_t i = 0; i < run; i++) in.push_back('\\');
      const size_t post = rng() % 5000;
      for (size_t i = 0; i < post; i++) in.push_back(uint8_t(a[rng() % alen]));
    } else if (kind == 1) {  // UTF-8 fragments at arbitrary offsets
      n += 4000;
      for (size_t i = 0; i < n; i++) in.push_back(uint8_t(rng() % 4 ? 'a' + rng() % 26 : a[rng() % alen]));
      const int k = 1 + int(rng() % 8);
      for (int j = 0; j < k; j++) {
        const char *f = utf8bits[rng() % 20];
        size_t pos = rng() % (in.size() + 1);
        if (rng() % 3 == 0) pos = (rng() % (in.size() / 128)) * 128 + (rng() % 7) - 3;
        if (rng() % 4 == 0) pos = (rng() % (in.size() / 4096 + 1)) * 4096 + (rng() % 7) - 3;
        if (pos > in.size()) pos = in.size();
        in.insert(in.begin() + long(pos), f, f + strlen(f));
      }
    } else if (kind == 2) {  // mostly valid multi-byte text
      n += 2000;
      while (in.size() < n) {
        const size_t pick[] = {0, 1, 2, 14, 15, 16, 17, 18, 19};
        const char *f = utf8bits[pick[rng() % 9]];
        if (rng() % 3) in.push_back(uint8_t(' ' + rng() % 90)); else in.insert(in.end(), f, f + strlen(f));
      }
      if (rng() % 2) in[rng() % in.size()] ^= uint8_t(1u << (rng() % 8));
      if (rng() % 4 == 0) in.resize(in.size() - rng() % 4);
    } else if (kind == 3) {  // several elements: the ticket pipeline, the chain and windows of the look-back
      n = 30000 + rng() % 400000;
      for (size_t i = 0; i < n; i++) in.push_back(uint8_t(rng() % 3 ? 'a' + rng() % 26 : a[rng() % alen]));
    } else if (kind == 4) {  // exact block / element multiples, truncated sequence at the very end
      n = (1 + rng() % 20) * 4096;
      if (rng() % 2) n = (1 + rng() % 3) * 32768;
      in.assign(n, 'a');
      for (int j = 0; j < 200; j++) in[rng() % in.size()] = uint8_t("\"\\ {}:,\n"[rng() % 8]);
      const char *tails[] = {"\xc3", "\xe2\x82", "\xf0\x9f\x98", "\xf0\x9f\x98\x80", "ab", "\xe2\x82\xac", "\\", "\\\"", "\"", "1"};
      const char *t = tails[rng() % 10];
      memcpy(in.data() + in.size() - strlen(t), t, strlen(t));
    } else if (kind == 5) {  // the document (or shard) starts inside a backslash run: launch carry-in meets boundary walks
      const size_t runs[] = {0, 1, 2, 3, 15, 16, 17, 31, 32, 33, 127, 129, 4095, 4096, 4097, 8192};
      const size_t long_runs[] = {32767, 32768, 32769, 36864};  // (slow under emulation: one rendezvous per 32 bytes walked)
      const size_t run = (rng() % 8 == 0) ? long_runs[rng() % 4] : runs[rng() % 16];
      for (size_t i = 0; i < run; i++) in.push_back('\\');
      if (rng() % 2) in.push_back('"');
      const size_t post = rng() % 3 ? rng() % 6000 : 0;
      for (size_t i = 0; i < post; i++) in.push_back(uint8_t(a[rng() % alen]));
      force_state = 1u | uint32_t(rng() % 8);
    } else {
      n += (rng() % 3) * 4096;
      for (size_t i = 0; i < n; i++) in.push_back(uint8_t(a[rng() % alen]));
    }
    if (in.empty()) in.push_back(' ');
    // (std::vector storage is 16-byte aligned with glibc malloc; assert it, the TMA path needs it)
    std::vector<uint8_t> buf0(in);
    if (reinterpret_cast<uintptr_t>(buf0.data()) & 15u) { fprintf(stderr, "unaligned vector storage\n"); return 3; }
    const unsigned grid = 1 + unsigned(rng() % 3);
    const uint32_t state_in = (force_state != 0xFFFFFFFFu) ? force_state : ((rng() % 3 == 0) ? uint32_t(rng() % 8) : 0u);
    check(cx, buf0, 0, state_in, 0, grid, true, "tma");
    if (it % 3 == 0) check(cx, buf0, 0, state_in, 1 + uint32_t(rng() % 3), grid, true, "chunked");
    if (it % 2 == 0) check_minify(cx, buf0, 0, (it % 6 == 0) ? 1 + uint32_t(rng() % 3) : 0, grid, it % 4 != 0, rng() % 17);
    if (it % 5 == 1 && buf0.size() > 3) check_minify(cx, buf0, 1 + rng() % 3, 0, grid, true, rng() % 17);
    if (kind == 1 || kind == 2 || kind == 4 || it % 3 == 0) {
      check_utf8v2(cx, buf0, 0, (it % 4 == 0) ? 1 + uint32_t(rng() % 2) : 0, grid, it % 5 != 0);
      if (it % 3 == 1 && buf0.size() > 3) check_utf8v2(cx, buf0, 1 + rng() % 3, 0, grid, true);
    }
    if (it % 4 == 1) check(cx, buf0, 0, state_in, 0, grid, false, "plain loads");
    if (it % 4 == 2 && buf0.size() > 3) check(cx, buf0, 1 + rng() % 3, state_in, 0, grid, true, "misaligned");
  }
  if (g_fail) { printf("FAILED\n"); return 1; }
  printf("simt emulation OK (%d cases)\n", iters);
  return 0;
}
