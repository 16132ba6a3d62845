// sjb200_fold.cpp -- the pure host folds of the sharded passes (sjb200_stream_fold, sjb200_delimited_fold) and the shard
// helpers of include/sjb200.h that need no device.  No CUDA: the CPU tests drive these through ctypes.
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "../../include/sjb200.h"
#include "sjb200_bits.cuh"
#include "sjb200_common.h"
#include "sjb200_params.h"

using namespace sjb200;

namespace {
enum : uint32_t { kRoleValue = 0, kRoleSep, kRoleOpenObj, kRoleCloseObj, kRoleOpenArr, kRoleCloseArr };  // as in sjb200_docs.cu
bool starts_document(uint32_t cur, uint32_t before) {  // find_next_document_index.h L60-88
  if (cur == kRoleSep || cur == kRoleCloseObj || cur == kRoleCloseArr) return false;
  return !(before == kRoleOpenObj || before == kRoleOpenArr || before == kRoleSep);
}
}  // namespace

// The fold of the summaries into the whole stream's finish() (json_structural_indexer.h L249-343, L395-396).  T = all
// structurals, n0 = T less the stream's last one when it ends inside a string (streaming modes).  The last document start
// g of [0, n0) is the last internal start of the last shard that has one, unless the first structural of a later shard
// starts a document across its cut; the brackets from g on are that shard's nets after its start plus the later shards'
// nets.  Then m = n0 when they balance, else g (0 without any start), as find_next_document_index.
extern "C" int sjb200_stream_fold(int mode, int nranks, uint32_t final_state, uint32_t flags_all, const sjb200_stream_summary *sums,
                                  sjb200_stream_fold_result *res, sjb200_stream_rank *ranks) {
  if (!res || !ranks || !sums || nranks < 1 || nranks > kMaxRanks || mode < SJB200_REGULAR || mode > SJB200_STREAMING_FINAL) return SJB200_UNEXPECTED_ERROR;
  memset(res, 0, sizeof(*res));
  memset(ranks, 0, sizeof(*ranks) * size_t(nranks));
  uint64_t base[kMaxRanks], off = 0, T = 0;
  int holder = -1;
  for (int r = 0; r < nranks; r++) {
    ranks[r].bytes_before = off;
    off += sums[r].len;
    base[r] = T;
    T += sums[r].count;
    if (sums[r].count) holder = r;
  }
  const uint64_t L = off;
  res->total_bytes = L;
  const bool streaming = mode != SJB200_REGULAR, unclosed = (final_state >> 1) & 1u;
  auto done = [&](int err) {
    res->error = err;
    for (int r = 0; r < nranks && res->n_written; r++) {
      const uint64_t k = res->n > base[r] ? res->n - base[r] : 0;
      ranks[r].kept = std::min<uint64_t>(k, sums[r].count);
    }
    for (int r = 0, prev = -1; r < nranks; r++) {  // prev: the last earlier shard with kept structurals
      if (ranks[r].kept == 0) continue;
      ranks[r].first_starts_document = (prev < 0) ? 1u : uint32_t(starts_document(sums[r].role_first, sums[prev].role_last));
      prev = r;
    }
    return err;
  };
  if (flags_all & kFlagInternal) return done(SJB200_UNEXPECTED_ERROR);
  if (streaming && L == 0) return done(SJB200_UTF8_ERROR);           // L198-204: nothing left after the trim
  if (!streaming && unclosed) return done(SJB200_UNCLOSED_STRING);   // L255-259
  if (flags_all & kFlagCtl) return done(SJB200_UNESCAPED_CHARS);    // L261-263
  res->n_written = 1;
  res->n = T;
  if (T == 0) return done(SJB200_EMPTY);                             // L289-291
  const bool utf8 = (flags_all & kFlagUtf8) != 0;
  if (!streaming) return done(utf8 ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
  const uint64_t n0 = T - (unclosed ? 1 : 0);
  if (mode == SJB200_STREAMING_PARTIAL && unclosed && n0 == 0) { res->n = 0; return done(SJB200_CAPACITY); }  // L298-302
  // the last document start g < n0 and the bracket balance of [g, n0); gv = global byte of structural g
  uint64_t g = 0, gv = 0;
  bool found = false;
  int64_t nobj = 0, narr = 0;
  for (int r = nranks - 1; r >= 0 && !found; r--) {
    const uint64_t kp = sums[r].count - ((unclosed && r == holder) ? 1 : 0);
    if (kp == 0) continue;
    nobj += sums[r].net_obj;
    narr += sums[r].net_arr;
    if (sums[r].has_start) {
      found = true; g = base[r] + sums[r].start_index; gv = ranks[r].bytes_before + sums[r].start_byte;
    } else if (base[r] > 0) {
      int q = r - 1;
      while (q >= 0 && sums[q].count == 0) q--;
      if (q >= 0 && starts_document(sums[r].role_first, sums[q].role_last)) { found = true; g = base[r]; gv = ranks[r].bytes_before + sums[r].first_byte; }
    }
  }
  if (!found && n0 > 0) {  // the start is structural 0
    int r0 = 0;
    while (sums[r0].count == 0) r0++;
    gv = ranks[r0].bytes_before + sums[r0].first_byte;
  }
  const uint64_t m = (n0 == 0) ? 0 : ((nobj == 0 && narr == 0) ? n0 : g);
  if (mode == SJB200_STREAMING_PARTIAL) {  // L303-317
    if (m == 0) {
      const bool idx0_zero = sums[0].count > 0 && sums[0].first_byte == 0;
      if (idx0_zero) { res->n = n0; return done(SJB200_CAPACITY); }
      res->n = 0;
      return done(SJB200_EMPTY);
    }
    res->n = m;
    return done(utf8 ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
  }
  // streaming final, L329-343: word m + 1 = old word m, word m = L; the ranks that hold them store them shard-relative
  uint64_t old_m;
  if (m >= T) old_m = L;                                                            // a sentinel
  else if (m == T - 1 && unclosed) old_m = ranks[holder].bytes_before + sums[holder].last_byte;  // the dropped quote
  else old_m = gv;                                                                  // a document start
  const uint64_t pos[2] = {m, m + 1}, val[2] = {L, old_m};
  for (int k = 0; k < 2; k++) {
    int r = nranks - 1;
    uint64_t local = sums[r].count + (pos[k] - T);
    if (pos[k] < T) {
      r = 0;
      while (!(pos[k] >= base[r] && pos[k] < base[r] + sums[r].count)) r++;
      local = pos[k] - base[r];
    }
    sjb200_stream_rank &w = ranks[r];
    w.rewrite_pos[w.nrewrites] = uint32_t(local);
    w.rewrite_val[w.nrewrites] = uint32_t(val[k] - w.bytes_before);
    w.nrewrites++;
  }
  res->n = m;
  if (m == 0) return done(SJB200_EMPTY);
  return done(utf8 ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
}

// The fold of a delimited pass's filter round into the whole stream's finish() for modes 3..6 (json_structural_indexer.h
// L344-396 with find_next_document_index_json_sequence / filter_comma_delimited, as filter_finish_kernel runs it on one
// GPU).  The filtered entries are sorted across the ranks, so the global last separator is the last one of the last
// rank that counted any, and the entries before it are the filtered entries of the ranks before plus its `below`.
// find_next_document_index over the first k filtered entries is sjb200_stream_fold's walk over the ranks' walk
// summaries (every rank's full walk, the last rank's walk_below when k ends at its `below`).  The words after n are those
// of the array the reference's in-place filter leaves: the filtered entries, then the scan's structurals, then the
// sentinels len, len, 0.
extern "C" int sjb200_delimited_fold(int mode, int nranks, uint32_t final_state, uint32_t flags_all, const sjb200_delimited_summary *sums,
                                     sjb200_delimited_fold_result *res, sjb200_delimited_rank *ranks) {
  if (!res || !ranks || !sums || nranks < 1 || nranks > kMaxRanks || mode < SJB200_JSON_SEQUENCE_PARTIAL || mode > SJB200_COMMA_DELIMITED_FINAL)
    return SJB200_UNEXPECTED_ERROR;
  memset(res, 0, sizeof(*res));
  memset(ranks, 0, sizeof(*ranks) * size_t(nranks));
  uint64_t base[kMaxRanks], off = 0, T = 0, W = 0, seps = 0;
  int sep_rank = -1;  // the last rank that counted a separator
  for (int r = 0; r < nranks; r++) {
    ranks[r].bytes_before = off;
    ranks[r].filtered_before = W;
    off += sums[r].len;
    base[r] = T;
    T += sums[r].count;
    W += sums[r].filtered;
    seps += sums[r].seps;
    if (sums[r].seps) sep_rank = r;
  }
  const uint64_t L = off;
  res->total_bytes = L;
  for (int k = 0; k < 3; k++) res->tail_rank[k] = -1;
  const bool rs = (mode == SJB200_JSON_SEQUENCE_PARTIAL || mode == SJB200_JSON_SEQUENCE_FINAL);
  const bool is_final = (mode == SJB200_JSON_SEQUENCE_FINAL || mode == SJB200_COMMA_DELIMITED_FINAL);
  const bool unclosed = (final_state >> 1) & 1u;
  auto word = [&](int k, uint64_t p) {  // word p of the array after the in-place filter -> tail k
    if (p < W || p < T) {
      const bool f = p < W;
      int r = 0;
      while (!(f ? (p >= ranks[r].filtered_before && p < ranks[r].filtered_before + sums[r].filtered) : (p >= base[r] && p < base[r] + sums[r].count))) r++;
      res->tail_rank[k] = r;
      res->tail_pos[k] = uint32_t(p - (f ? ranks[r].filtered_before : base[r]));
      res->tail_filtered[k] = f ? 1u : 0u;
    } else {
      res->tail_val[k] = p < T + 2 ? uint32_t(L) : 0u;
    }
  };
  auto words_from = [&](uint64_t p) { for (int k = 0; k < 3; k++) word(k, p + uint64_t(k)); };
  auto done = [&](int err) {
    res->error = err;
    for (int r = 0; r < nranks && res->n_written; r++) {
      const uint64_t k = res->n > ranks[r].filtered_before ? res->n - ranks[r].filtered_before : 0;
      ranks[r].kept = std::min<uint64_t>(k, sums[r].filtered);
    }
    for (int r = 0, prev = -1; r < nranks; r++) {  // prev: the last earlier shard with kept entries
      if (ranks[r].kept == 0) continue;
      ranks[r].first_starts_document = (prev < 0) ? 1u : uint32_t(starts_document(sums[r].walk.role_first, sums[prev].walk.role_last));
      prev = r;
    }
    return err;
  };
  // find_next_document_index over the first k filtered entries
  auto walk = [&](uint64_t k) -> uint64_t {
    sjb200_stream_summary ws[kMaxRanks];
    for (int r = 0; r < nranks; r++) {
      const uint64_t fb = ranks[r].filtered_before;
      const uint64_t cnt = std::min<uint64_t>(k > fb ? k - fb : 0, sums[r].filtered);
      if (cnt == 0) memset(&ws[r], 0, sizeof(ws[r]));
      else ws[r] = (cnt == sums[r].filtered) ? sums[r].walk : sums[r].walk_below;
      ws[r].count = cnt;
      ws[r].len = sums[r].len;
    }
    sjb200_stream_fold_result fr;
    sjb200_stream_rank fk[kMaxRanks];
    sjb200_stream_fold(SJB200_STREAMING_FINAL, nranks, 0, 0, ws, &fr, fk);
    return fr.n;
  };
  if (flags_all & kFlagInternal) return done(SJB200_UNEXPECTED_ERROR);
  if (L == 0) return done(SJB200_UTF8_ERROR);                        // L198-204: nothing left after the trim
  if (flags_all & kFlagCtl) return done(SJB200_UNESCAPED_CHARS);    // L261-263
  res->n_written = 1;
  res->n = T;
  if (T == 0) { words_from(0); return done(SJB200_EMPTY); }          // L289-291
  if (!is_final && unclosed && T == 1) { res->n = 0; words_from(0); return done(SJB200_CAPACITY); }  // L298-302, before the filter
  uint64_t m = 0, n_res = W, next_start = L;
  bool too_large = false;
  const uint64_t last_sep = sep_rank >= 0 ? ranks[sep_rank].bytes_before + sums[sep_rank].last_sep : 0;
  const uint64_t before_sep = sep_rank >= 0 ? ranks[sep_rank].filtered_before + sums[sep_rank].below : 0;
  if (W != 0) {
    if (rs) {
      if (seps == 0) m = is_final ? walk(W) : 0;
      else if (is_final) m = W;
      else {
        next_start = last_sep;
        if (seps < 2) too_large = true;
        else m = before_sep;
      }
    } else {
      if (is_final) m = walk(W);
      else if (seps == 0) too_large = true;
      else {
        next_start = last_sep + 1;
        if (before_sep != 0) { n_res = before_sep; m = walk(before_sep); }
      }
    }
  }
  if (!is_final) {  // L344-359, L367-384
    if (too_large) { res->n = n_res; words_from(n_res); return done(SJB200_CAPACITY); }
    if (m == 0) { res->n = 0; words_from(0); return done(SJB200_EMPTY); }
    res->n = m;
    res->tail_val[0] = uint32_t(next_start);
    word(1, m + 1);
    word(2, m + 2);
  } else {  // L360-366, L385-393: word m + 1 = the old word m
    res->n = m;
    res->tail_val[0] = uint32_t(L);
    word(1, m);
    word(2, m + 2);
    if (m == 0) return done(SJB200_EMPTY);
  }
  return done((flags_all & kFlagUtf8) ? SJB200_UTF8_ERROR : SJB200_SUCCESS);
}

extern "C" uint32_t sjb200_fold_state(const uint32_t *ttables, int nshards_before) {
  uint32_t state = 0;
  for (int i = 0; i < nshards_before; i++) state = tt_apply(ttables[i], state);
  return state;
}

extern "C" size_t sjb200_shard_cut(const uint8_t *buf, size_t len, size_t nominal) {
  if (nominal >= len) return len;
  size_t cut = nominal;
  for (int k = 0; k < 3 && cut > 0 && (buf[cut] & 0xC0) == 0x80; k++) cut--;
  return cut;
}

extern "C" size_t sjb200_shard_cut_line(const uint8_t *buf, size_t len, size_t nominal, size_t window) {
  if (nominal >= len) return len;
  const size_t lo = nominal > window ? nominal - window : 0;
  for (size_t cut = nominal; cut > lo; cut--)
    if (buf[cut - 1] == 0x0A) return cut;
  return sjb200_shard_cut(buf, len, nominal);
}

// ---- sharded grammar (sjb200_document_errors_sharded)
namespace {
constexpr uint32_t kEdgeFailed = 1, kEdgeBadTable = 2, kEdgeWhole = 4, kEdgeFirstStarts = 8, kEdgeLastStarts = 16;
uint32_t type_byte(uint32_t types, int b) { return (types >> (8 * b)) & 0xFFu; }
}  // namespace

// The edge round: every rank's place in the stream and the halo of its structurals.  A rank's neighbours k - 2, k - 1
// and k + 1 may lie on any other rank, past ranks with n = 0 or 1.
extern "C" int sjb200_grammar_edge_fold(int nranks, const sjb200_grammar_edge *e, sjb200_grammar_edge_fold_result *res, sjb200_grammar_rank *ranks) {
  if (!e || !res || !ranks || nranks < 1 || nranks > kMaxRanks) return SJB200_UNEXPECTED_ERROR;
  memset(res, 0, sizeof(*res));
  memset(ranks, 0, sizeof(*ranks) * size_t(nranks));
  bool failed = false, capacity = false, differ = false;
  const bool whole = (e[0].flags & kEdgeWhole) != 0;
  for (int r = 0; r < nranks; r++) {
    failed = failed || (e[r].flags & kEdgeFailed);
    capacity = capacity || e[r].max_depth == 0 || e[r].max_depth > SJB200_DOCUMENT_MAX_DEPTH;
    differ = differ || e[r].max_depth != e[0].max_depth || ((e[r].flags & kEdgeWhole) != 0) != whole;
    if (!whole && (e[r].flags & kEdgeBadTable)) res->bad_table = 1;
  }
  res->error = failed ? SJB200_UNEXPECTED_ERROR : capacity ? SJB200_CAPACITY : differ ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
  uint64_t tokens = 0, docs = 0;
  for (int r = 0; r < nranks; r++) {
    sjb200_grammar_rank &k = ranks[r];
    k.tokens_before = tokens;
    k.docs_before = docs;
    k.owned = whole ? (r == 0 ? 1u : 0u) : e[r].ndocs;
    k.holds_root = tokens == 0 && e[r].n > 0;
    tokens += e[r].n;
    docs += k.owned;
  }
  res->n = tokens;
  res->ndocs = docs;
  // does rank q's structural j (0 or n - 1) start a document
  auto starts = [&](int q, bool last) {
    if (ranks[q].holds_root && (!last || e[q].n == 1)) return true;
    return !whole && (e[q].flags & (last ? kEdgeLastStarts : kEdgeFirstStarts)) != 0;
  };
  uint32_t last_type = 0xFFu;
  for (int r = 0; r < nranks; r++)
    if (e[r].n) last_type = type_byte(e[r].types, 3);
  for (int r = 0; r < nranks; r++) {
    sjb200_grammar_rank &k = ranks[r];
    uint32_t before[2] = {0xFFu, 0xFFu};  // [0] the structural just before, [1] the one before it
    int got = 0, prev = -1;
    for (int q = r - 1; q >= 0 && got < 2; q--) {
      if (!e[q].n) continue;
      if (prev < 0) prev = q;
      before[got++] = type_byte(e[q].types, 3);
      if (got < 2 && e[q].n >= 2) before[got++] = type_byte(e[q].types, 2);
    }
    int next = -1;
    for (int q = r + 1; q < nranks && next < 0; q++)
      if (e[q].n) next = q;
    k.halo_before = before[1] | (before[0] << 8) | 0xFFFF0000u;
    k.halo_after = next < 0 ? 0xFFu : type_byte(e[next].types, 0);
    k.halo_flags = (prev >= 0 && starts(prev, true) ? 1u : 0u) | (next >= 0 && starts(next, false) ? 2u : 0u) | (k.holds_root ? 4u : 0u);
    k.last_type = last_type;
  }
  return res->error;
}

// The result round: a document that spans ranks is owned by the rank it starts on, and its error is the first in rank
// order over the ranks it spans -- its owner's own, then the leading segments of the ranks up to the next start.
extern "C" int sjb200_grammar_result_fold(int nranks, const sjb200_grammar_edge *e, const sjb200_grammar_tally *t,
                                          sjb200_sharded_document_errors_result *out, sjb200_sharded_document_error *last) {
  if (!e || !t || !out || !last || nranks < 1 || nranks > kMaxRanks) return SJB200_UNEXPECTED_ERROR;
  sjb200_grammar_edge_fold_result res;
  sjb200_grammar_rank ranks[kMaxRanks];
  sjb200_grammar_edge_fold(nranks, e, &res, ranks);
  const bool whole = (e[0].flags & kEdgeWhole) != 0;
  const uint64_t none = ~0ull;
  uint64_t key[kMaxRanks];
  int owner = -1;
  for (int r = 0; r < nranks; r++) {
    if (owner >= 0 && t[r].lead < key[owner]) key[owner] = t[r].lead;
    if (ranks[r].owned) {
      owner = r;
      key[r] = t[r].last;
    }
  }
  if (whole && res.n == 0) key[0] = uint64_t(SJB200_EMPTY);  // {EMPTY, 0}
  out->error = SJB200_SUCCESS;
  out->first_error = SJB200_SUCCESS;
  out->ndocs = res.ndocs;
  out->ndocs_in_error = 0;
  out->first_doc_in_error = none;
  out->first_error_index = none;
  for (int r = 0; r < nranks; r++) {
    if (!ranks[r].owned) continue;
    uint64_t next = res.n;  // one past the last document's value when it is good: the next document's start
    for (int q = r + 1; q < nranks && !whole; q++)
      if (ranks[q].owned) { next = ranks[q].tokens_before + e[q].first_start; break; }
    last[r].error = key[r] == none ? 0 : int32_t(key[r] & 0xFFu);
    last[r].reserved = 0;
    last[r].index = key[r] == none ? next : key[r] >> 8;
    out->ndocs_in_error += t[r].errors + (key[r] != none ? 1u : 0u);
    if (out->first_doc_in_error != none) continue;
    if (t[r].first_doc != 0xFFFFFFFFu) {
      out->first_doc_in_error = ranks[r].docs_before + t[r].first_doc;
      out->first_error = int32_t(t[r].first_key & 0xFFu);
      out->first_error_index = t[r].first_key >> 8;
    } else if (key[r] != none) {
      out->first_doc_in_error = ranks[r].docs_before + ranks[r].owned - 1;
      out->first_error = last[r].error;
      out->first_error_index = last[r].index;
    }
  }
  return out->error;
}

// ---- sharded JSON Pointer lookup (sjb200_at_pointer_sharded)
// The edge round: every rank's place in the stream, the ranks its walks are handed between, and for the document that
// holds its last structural (its tail document): whether it goes on past the rank, how many structurals it has on later
// ranks, and the first token in error of those pieces.  A document's piece on a later rank is that rank's leading
// segment (all of its structurals when it has no table entry); ranks with 0 structurals hold no piece.  The bases, the
// ownership and the type after a rank's last structural are the grammar's edge fold.
extern "C" int sjb200_pointer_edge_fold(int nranks, const sjb200_pointer_edge *e, sjb200_pointer_edge_fold_result *res, sjb200_pointer_rank *ranks) {
  if (!e || !res || !ranks || nranks < 1 || nranks > kMaxRanks) return SJB200_UNEXPECTED_ERROR;
  memset(res, 0, sizeof(*res));
  memset(ranks, 0, sizeof(*ranks) * size_t(nranks));
  const bool whole = (e[0].flags & kPtrEdgeWhole) != 0;
  sjb200_grammar_edge ge[kMaxRanks];
  bool failed = false, over = false, differ = false;
  for (int r = 0; r < nranks; r++) {
    failed = failed || (e[r].flags & kPtrEdgeFailed);
    over = over || (e[r].flags & kPtrEdgeOver) || e[r].npointers > uint32_t(kPtrMaxPointers);
    differ = differ || ((e[r].flags & kPtrEdgeWhole) != 0) != whole || e[r].npointers != e[0].npointers || e[r].hash != e[0].hash;
    if (!whole && (e[r].flags & kPtrEdgeBadTable)) res->bad_table = 1;
    const uint32_t t0 = e[r].types & 0xFFu, t1 = (e[r].types >> 8) & 0xFFu;
    ge[r] = sjb200_grammar_edge{e[r].n, whole ? 0u : e[r].ndocs, (e[r].flags & kPtrEdgeWhole) ? uint32_t(kGramEdgeWhole) : 0u, 1u,
                                t0 | 0xFFFF00u | (t1 << 24), e[r].first_entry};
  }
  sjb200_grammar_edge_fold_result gres;
  sjb200_grammar_rank g[kMaxRanks];
  sjb200_grammar_edge_fold(nranks, ge, &gres, g);
  over = over || gres.n > 0xFFFFFFFCull;  // kSuspend, kNone and every index a walk reaches must stay apart in 32 bits
  res->n = gres.n;
  res->ndocs = gres.ndocs;
  res->error = failed ? SJB200_UNEXPECTED_ERROR : over ? SJB200_CAPACITY : differ ? SJB200_UNEXPECTED_ERROR : SJB200_SUCCESS;
  // the leading segment of rank r: [0, lead_end(r)); a table entry at 0 leaves it empty
  auto lead_end = [&](int r) { return (whole || !e[r].ndocs) ? e[r].n : e[r].first_entry; };
  int open_owner = -1, prev = -1;  // the owner of the document the structurals so far end in; the last holder
  for (int r = 0; r < nranks; r++) {
    sjb200_pointer_rank &k = ranks[r];
    k.tokens_before = g[r].tokens_before;
    k.docs_before = g[r].docs_before;
    k.owned = g[r].owned;
    k.next_type = g[r].halo_after;
    k.prev_holder = prev;
    k.next_holder = -1;
    for (int q = r + 1; q < nranks && k.next_holder < 0; q++)
      if (e[q].n) k.next_holder = q;
    k.lead_owner = k.tail_owner = k.tail_through = -1;
    k.tail_error_index = ~0ull;
    if (!e[r].n) continue;
    if (whole) {
      k.walks = open_owner < 0 ? 1u : 0u;  // the first holder walks from the root
      k.lead_owner = open_owner;
      open_owner = 0;
    } else {
      k.walks = e[r].ndocs;
      k.lead_owner = lead_end(r) > 0 ? open_owner : -1;
      if (e[r].ndocs) open_owner = r;
    }
    k.tail_owner = open_owner;
    prev = r;
  }
  for (int r = 0; r < nranks; r++) {
    sjb200_pointer_rank &k = ranks[r];
    if (!e[r].n || k.tail_owner < 0) continue;
    for (int q = k.next_holder; q >= 0 && q < nranks; q++) {
      if (!e[q].n) continue;
      const uint32_t le = lead_end(q);
      if (le == 0) break;  // a document starts at q's structural 0
      k.tail_continues = 1;
      k.tail_through = q;
      k.tail_after += le;
      if (!k.tail_error && e[q].lead_error_index != 0xFFFFFFFFu) {
        k.tail_error = e[q].lead_error;
        k.tail_error_index = g[q].tokens_before + e[q].lead_error_index;
      }
      if (le < e[q].n) break;  // the document ends on q
    }
  }
  return res->error;
}
