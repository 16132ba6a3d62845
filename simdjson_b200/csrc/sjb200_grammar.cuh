// sjb200_grammar.cuh -- the nesting grammar of stage 2 over the stage-2-lite tokens (sjb200_document_errors_dev): the
// error json_iterator::walk_document (src/generic/stage2/json_iterator.h L120-244) returns for every document of a stream,
// decided for every structural at once.  Written against sjb200_simt.cuh so that the host SIMT emulation
// (tests/grammar_emul.cpp) runs the same source as the sm_90a kernels in sjb200_grammar.cu.
//
// Given the document's prefix before structural k is valid, what the walk expects at k follows from the types at k-2 and
// k-1 and from c(k), the kind of the innermost open container; the depth D(k) is a prefix sum of +1 (opener) / -1
// (closer), where an empty pair `{}` / `[]` counts as one scalar.  The first error of a document is the error at the
// smallest k, so each k is judged alone as if its prefix were valid, and the smallest judged error wins.
//
// Tiles are kTile consecutive structurals, one warp each, independent of document boundaries; a document start resets
// the depth.  c(k) is the opener of the last structural before k whose depth is below D(k): inside the tile a lane keeps
// the openers it opened itself and otherwise searches the tile's earlier lanes; for a container opened before the tile
// it reads the tile's incoming stack.  The incoming stacks come from per-tile stack records (pass A: the closers a tile
// pops below its start, the kinds of the openers still open at its end), folded in document order by a fan-out-32
// tree (pass B: fold_up, fold_down).  A record holds at most `words` * 32 kinds: anything deeper is already a
// DEPTH_ERROR of its document.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "sjb200_params.h"
#include "sjb200_simt.cuh"

namespace sjb200 {
namespace gram {

// simdjson::error_code values (include/simdjson/error.h L19-54)
constexpr uint32_t kTapeError = 3, kDepthError = 4, kStringError = 5, kNumberError = 9, kEmpty = 13, kUnexpected = 24;
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr uint32_t kMaxDepth = 4096;  // SJB200_DOCUMENT_MAX_DEPTH
constexpr uint32_t kMaxWords = kMaxDepth / 32;
constexpr uint32_t kReset = 0x80000000u;  // record word 0: the record starts at a document start
constexpr uint32_t kPopsMask = 0x7FFFFFFFu;

struct DocError {  // sjb200_document_error
  int32_t error;
  uint32_t index;
};

struct Grammar {
  const uint8_t *type;      // sjb200_tokens_dev d_type
  const uint64_t *payload;  // ... d_payload
  uint32_t n;
  const uint32_t *starts;   // bit k: a document starts at structural k (bit 0 always set)
  bool whole;               // no table: one document [0, n), with the root-bracket check
  uint32_t max_depth;
  uint32_t words;           // kinds per record / 32: ceil(max_depth / 32)
  const uint32_t *prefix;   // per tile: the record of everything before it in its document (2 + words each)
};

SJ_DEV bool is_open(uint32_t t) { return t == '{' || t == '['; }
SJ_DEV bool is_close(uint32_t t) { return t == '}' || t == ']'; }
SJ_DEV bool is_scalar(uint32_t t) { return t == '"' || t == 'l' || t == 'u' || t == 'd' || t == 't' || t == 'f' || t == 'n'; }
SJ_DEV uint32_t closer_of(uint32_t t) { return t == '{' ? '}' : ']'; }
SJ_DEV bool start_at(const uint32_t *starts, uint32_t k) { return (sj_ldg_u32(starts + (k >> 5)) >> (k & 31u)) & 1u; }

// What lies around the structurals [0, n) of a Grammar.  NoHalo: nothing -- the whole stream (sjb200_document_errors_dev);
// the tile routines then do exactly what they did before halos existed.  ShardHalo: one rank's shard of a sharded pass
// (sjb200_document_errors_sharded): the neighbours of its first and last structurals, which may lie on any other rank.
struct NoHalo {
  SJ_DEV uint8_t type_outside(const Grammar &, uint32_t) const { return 0xFF; }
  SJ_DEV bool pair_across(const Grammar &, uint32_t, bool) const { return false; }
  SJ_DEV bool start_before(const Grammar &g, uint32_t k) const { return start_at(g.starts, k - 1); }
  SJ_DEV bool ends_at(const Grammar &, uint32_t) const { return true; }
  SJ_DEV uint32_t last_type(const Grammar &g) const { return g.whole ? sj_ldg_u8(g.type + g.n - 1) : 0u; }
  SJ_DEV bool root_at(uint32_t k) const { return k == 0; }
};

struct ShardHalo {
  static constexpr uint32_t kPrevStart = 1, kNextStart = 2, kRoot = 4;
  uint32_t before;  // types of the two structurals before structural 0: byte 0 the one two before, byte 1 the one just before (0xFF: none)
  uint32_t after;   // type of the structural after n - 1 (0xFF: none)
  uint32_t flags;   // kPrevStart: the structural before 0 starts a document; kNextStart: the one after n - 1 does; kRoot: 0 is the stream's first
  uint32_t last;    // whole mode: type of the stream's last structural
  // type of tile slot p = k + 2 outside [0, n): the halo before (p < 2) or after (p == n + 2)
  SJ_DEV uint8_t type_outside(const Grammar &g, uint32_t p) const {
    if (p < 2) return uint8_t(before >> (8u * p));
    return uint64_t(p) == uint64_t(g.n) + 2 ? uint8_t(after) : uint8_t(0xFF);
  }
  // an opener at n - 1 and the closer after the cut are an empty pair (closes: that closer matches the opener)
  SJ_DEV bool pair_across(const Grammar &g, uint32_t k, bool closes) const { return k + 1 == g.n && closes && !(flags & kNextStart); }
  SJ_DEV bool start_before(const Grammar &g, uint32_t k) const { return k ? start_at(g.starts, k - 1) : (flags & kPrevStart) != 0; }
  // false when structural n - 1 looks like a document's end only because the shard ends there
  SJ_DEV bool ends_at(const Grammar &g, uint32_t k) const { return k + 1 != g.n || after == 0xFFu || (flags & kNextStart) != 0; }
  SJ_DEV uint32_t last_type(const Grammar &) const { return last; }
  SJ_DEV bool root_at(uint32_t k) const { return k == 0 && (flags & kRoot) != 0; }
};

// A tile's structurals in shared memory: ty[i + 2] = type of structural tile0 + i (halo: two before, one after; past the
// ends the halo's types, 0xFF without one), dep[i] = its depth D before it, lane_min[l] = the lowest depth among lane l's structurals.
template <int ITEMS>
struct TileSmem {
  static constexpr uint32_t kTile = 32u * ITEMS;
  uint8_t ty[kTile + 4];
  int32_t dep[kTile];
  int32_t lane_min[32];
  uint32_t rec[2 + kMaxWords];  // pass A: the record being built; pass B: the running fold
  uint32_t child[2 + kMaxWords];
};

// The tile's types, and per structural its depth change: +1 a non-empty opener, -1 a closer that does not end an empty
// pair.  An empty pair is an opener followed, in the same document, by its own closer.
template <int ITEMS, class H = NoHalo>
SJ_DEV void load_tile(const Grammar &g, TileSmem<ITEMS> &sm, unsigned lane, uint32_t tile0, const H &h = H()) {
  for (uint32_t i = lane; i < TileSmem<ITEMS>::kTile + 3; i += 32) {
    const uint64_t k = uint64_t(tile0) + i - 2;  // wraps below 0: past the end too
    sm.ty[i] = uint64_t(tile0) + i >= 2 && k < g.n ? uint8_t(sj_ldg_u8(g.type + k)) : h.type_outside(g, tile0 + i);
  }
  sj_syncwarp();
}

template <int ITEMS, class H = NoHalo>
SJ_DEV int delta_at(const Grammar &g, const TileSmem<ITEMS> &sm, uint32_t tile0, uint32_t i, const H &h = H()) {
  const uint32_t t = sm.ty[i + 2], k = tile0 + i;
  if (is_open(t)) {
    const bool empty = (k + 1 < g.n && sm.ty[i + 3] == closer_of(t) && !start_at(g.starts, k + 1)) || h.pair_across(g, k, sm.ty[i + 3] == closer_of(t));
    return empty ? 0 : 1;
  }
  if (is_close(t)) {
    const bool empty = !start_at(g.starts, k) && sm.ty[i + 1] == (t == '}' ? '{' : '[');
    return empty ? 0 : -1;
  }
  return 0;
}

// Segmented depths of the tile: dep[i] = depth before structural tile0 + i, counted from the tile start for the
// structurals before the tile's first document start, from that start (0) after it.  Returns the tile's first document
// start (kNone: none) in *first_reset and its last in *last_reset.
template <int ITEMS, class H = NoHalo>
SJ_DEV void tile_depths(const Grammar &g, TileSmem<ITEMS> &sm, unsigned lane, uint32_t tile0, uint32_t *first_reset, uint32_t *last_reset,
                        const H &h = H()) {
  const uint32_t i0 = lane * ITEMS;
  int d = 0;
  bool reset = false;
  uint32_t fr = kNone, lr = kNone;
  for (int j = 0; j < ITEMS; j++) {
    const uint32_t i = i0 + j, k = tile0 + i;
    if (k >= g.n) break;
    if (start_at(g.starts, k)) {
      reset = true;
      d = 0;
      if (fr == kNone) fr = k;
      lr = k;
    }
    sm.dep[i] = d;
    d += delta_at(g, sm, tile0, i, h);
  }
  // segmented exclusive scan over lanes of (reset, sum)
  uint32_t f = reset ? 1u : 0u;
  int v = d;
  for (int s = 1; s < 32; s <<= 1) {
    const uint32_t fu = sj_shfl_up(f, s);
    const int vu = int(sj_shfl_up(uint32_t(v), s));
    if (int(lane) >= s) {
      if (!f) v += vu;
      f |= fu;
    }
  }
  int inc = int(sj_shfl_up(uint32_t(v), 1));
  if (lane == 0) inc = 0;
  for (int j = 0; j < ITEMS; j++) {
    const uint32_t i = i0 + j, k = tile0 + i;
    if (k >= g.n || start_at(g.starts, k)) break;
    sm.dep[i] += inc;
  }
  *first_reset = sj_reduce_min(fr);
  const uint32_t l = sj_reduce_max(lr == kNone ? 0u : lr + 1u);
  *last_reset = l == 0 ? kNone : l - 1u;
  sj_syncwarp();
}

// ---- pass A: the tile's stack record (of its last document segment)
template <int ITEMS, class H = NoHalo>
SJ_DEV void tile_record(const Grammar &g, TileSmem<ITEMS> &sm, unsigned lane, uint32_t tile0, uint32_t *out, const H &h = H()) {
  uint32_t fr, lr;
  tile_depths<ITEMS>(g, sm, lane, tile0, &fr, &lr, h);
  const uint32_t seg0 = lr == kNone ? tile0 : lr;  // the last segment
  const uint32_t i0 = lane * ITEMS;
  const uint32_t cap = g.words * 32u;
  for (uint32_t w = lane; w < g.words; w += 32) sm.rec[2 + w] = 0;
  // depth after each structural: its minimum over the segment and over each lane's part
  int lmin = 0x7FFFFFFF, last_after = 0x80000000;
  for (int j = 0; j < ITEMS; j++) {
    const uint32_t i = i0 + j, k = tile0 + i;
    if (k >= g.n) break;
    if (k < seg0) continue;
    const int a = sm.dep[i] + delta_at(g, sm, tile0, i, h);
    lmin = a < lmin ? a : lmin;
    last_after = a;
  }
  const int seg_min = int(sj_reduce_min(uint32_t(lmin) ^ 0x80000000u) ^ 0x80000000u);  // signed order
  const int m = seg_min < 0 ? seg_min : 0;
  // the lane of the tile's last structural holds the end depth
  const uint32_t last_k = (uint64_t(tile0) + TileSmem<ITEMS>::kTile < g.n ? tile0 + TileSmem<ITEMS>::kTile : g.n) - 1u;
  const unsigned last_lane = (last_k - tile0) / ITEMS;
  const int end_depth = int(sj_shfl(uint32_t(last_after), int(last_lane)));
  // suffix minimum of the depth after, over the lanes after this one
  int sfx = lmin;
  for (int s = 1; s < 32; s <<= 1) {
    const int u = int(sj_shfl_down(uint32_t(sfx), s));
    if (lane + s < 32) sfx = u < sfx ? u : sfx;
  }
  int after_me = int(sj_shfl_down(uint32_t(sfx), 1));
  if (lane == 31) after_me = 0x7FFFFFFF;
  sj_syncwarp();
  // openers still open at the end: no later structural of the segment goes below their depth
  int run = after_me;
  for (int j = ITEMS - 1; j >= 0; j--) {
    const uint32_t i = i0 + j, k = tile0 + i;
    if (k >= g.n || k < seg0) continue;
    const int dl = delta_at(g, sm, tile0, i, h);
    const int a = sm.dep[i] + dl;
    if (dl == 1 && run >= a) {
      const uint32_t slot = uint32_t(a - m - 1);
      if (slot < cap && sm.ty[i + 2] == '[') sj_atomic_or(&sm.rec[2 + (slot >> 5)], 1u << (slot & 31u));
    }
    run = a < run ? a : run;
  }
  sj_syncwarp();
  const uint32_t cnt = uint32_t(end_depth - m);
  const uint32_t pops = uint32_t(-m) > kPopsMask ? kPopsMask : uint32_t(-m);
  const uint32_t c = cnt < cap ? cnt : cap;
  if (lane == 0) {
    out[0] = (lr != kNone ? kReset : 0u) | pops;
    out[1] = c;
  }
  for (uint32_t w = lane; w < (c + 31) / 32; w += 32) out[2 + w] = sm.rec[2 + w];
  sj_syncwarp();
}

// ---- pass B: records folded in order.  acc := acc then ch (both in shared memory, 2 + words each).
SJ_DEV void compose(unsigned lane, uint32_t *acc, const uint32_t *ch, uint32_t words) {
  const uint32_t ah = acc[0], ac = acc[1], bh = ch[0], bc = ch[1];
  const uint32_t bpops = bh & kPopsMask;
  const uint32_t cap = words * 32u;
  sj_syncwarp();
  if ((bh & kReset) || bpops >= ac) {
    for (uint32_t w = lane; w < (bc + 31) / 32; w += 32) acc[2 + w] = ch[2 + w];
    if (lane == 0) {
      if (bh & kReset) {
        acc[0] = bh;
      } else {
        const uint64_t p = uint64_t(ah & kPopsMask) + (bpops - ac);
        acc[0] = (ah & kReset) | (p > kPopsMask ? kPopsMask : uint32_t(p));
      }
      acc[1] = bc;
    }
  } else {
    const uint32_t m = ac - bpops;
    const uint32_t nc = m + bc < cap ? m + bc : cap;
    for (uint32_t w = (m >> 5) + lane; w < (nc + 31) / 32; w += 32) {
      const int off = int(w * 32u) - int(m);  // bit w*32 of acc is bit `off` of ch
      uint32_t v;
      if (off < 0) {
        const uint32_t keep = (1u << (m & 31u)) - 1u;
        v = (acc[2 + w] & keep) | (ch[2] << (m & 31u));
      } else {
        const uint32_t q = uint32_t(off) >> 5, s = uint32_t(off) & 31u;
        const uint32_t lo = ch[2 + q], hi = q + 1 < words ? ch[2 + q + 1] : 0u;
        v = s ? ((lo >> s) | (hi << (32u - s))) : lo;
      }
      acc[2 + w] = v;
    }
    if (lane == 0) acc[1] = nc;
  }
  sj_syncwarp();
}

// the words of a record in use: its header and its cnt kinds
SJ_DEV void copy_record(unsigned lane, uint32_t *dst, const uint32_t *src) {
  const uint32_t c = src[1];
  if (lane < 2) dst[lane] = src[lane];
  for (uint32_t w = lane; w < (c + 31) / 32; w += 32) dst[2 + w] = src[2 + w];
  sj_syncwarp();
}

// group g of up to 32 consecutive records of `level` (count of them): its fold into up[g]
SJ_DEV void fold_up_group(unsigned lane, uint32_t *acc, uint32_t *ch, const uint32_t *level, uint32_t count, uint32_t *up, uint32_t g, uint32_t words) {
  const size_t stride = 2 + words;
  if (lane < 2) acc[lane] = 0;
  sj_syncwarp();
  for (uint32_t c = g * 32; c < count && c < g * 32 + 32; c++) {
    copy_record(lane, ch, level + c * stride);
    compose(lane, acc, ch, words);
  }
  copy_record(lane, up + g * stride, acc);
}

// group g: its records of `level` replaced, in place, by the fold of everything before each in its document, starting
// from the group's own (up[g], already replaced the same way)
SJ_DEV void fold_down_group(unsigned lane, uint32_t *acc, uint32_t *ch, uint32_t *level, uint32_t count, const uint32_t *up, uint32_t g, uint32_t words) {
  const size_t stride = 2 + words;
  copy_record(lane, acc, up + g * stride);
  for (uint32_t c = g * 32; c < count && c < g * 32 + 32; c++) {
    copy_record(lane, ch, level + c * stride);
    copy_record(lane, level + c * stride, acc);
    compose(lane, acc, ch, words);
  }
}

// ---- pass C: the judgement of every structural of the tile
enum : uint32_t { kExpRoot, kExpValue, kExpKey, kExpColon, kExpAfter, kExpDone };

// the error of a value / root token at structural k of type t (0: none).  Inside a container every byte below '0' takes
// the number path (json_iterator.h L342), so a ',' there is a NUMBER_ERROR; the root's switch (L309-336) says TAPE_ERROR.
SJ_DEV uint32_t value_error(const Grammar &g, uint32_t k, uint32_t t, bool empty, int depth, bool root) {
  if (is_scalar(t)) return 0;
  if (t == 0) return uint32_t(g.payload[k] & 0xFFu);
  if (t == ',' && !root) return kNumberError;
  if (is_open(t)) return (!empty && depth + 1 >= int(g.max_depth)) ? kDepthError : 0u;
  return kTapeError;
}

// The first error of each document of the tile, as each lane sees it: report(pos, code, index) once per lane and document
// segment, pos a structural of the document (index is one past it for a document that ends too early).
template <int ITEMS, class F, class H = NoHalo>
SJ_DEV void tile_check(const Grammar &g, TileSmem<ITEMS> &sm, unsigned lane, uint32_t tile0, uint32_t tile, F &&report, const H &h = H()) {
  uint32_t fr, lr;
  tile_depths<ITEMS>(g, sm, lane, tile0, &fr, &lr, h);
  const uint32_t *pre = g.prefix + size_t(tile) * (2 + g.words);
  const uint32_t d_in = pre[1];
  const uint32_t i0 = lane * ITEMS;
  int lmin = 0x7FFFFFFF;
  for (int j = 0; j < ITEMS; j++) {
    const uint32_t i = i0 + j, k = tile0 + i;
    if (k >= g.n) break;
    if (k < fr) sm.dep[i] += int(d_in);
    lmin = sm.dep[i] < lmin ? sm.dep[i] : lmin;
  }
  sm.lane_min[lane] = lmin;
  // the lowest depth in the lanes before this one: a container opened below it is searched in the incoming stack at once
  int below = lmin;
  for (int s = 1; s < 32; s <<= 1) {
    const int u = int(sj_shfl_up(uint32_t(below), s));
    if (int(lane) >= s) below = u < below ? u : below;
  }
  int before_min = int(sj_shfl_up(uint32_t(below), 1));
  if (lane == 0) before_min = 0x7FFFFFFF;
  sj_syncwarp();
  const uint32_t last_type = h.last_type(g);
  // the lane's own open containers (bit: '['), and one cached answer from below the lane
  uint32_t lbits = 0, lcnt = 0;
  int ext_level = -1;
  uint32_t ext_kind = 0;
  // the lane's first error in the current document: its code, the structural it belongs to, the index it reports
  uint32_t seg_err = kNone, seg_pos = kNone, seg_idx = kNone;
  // the kind of the innermost container open at structural i of the tile, at depth L ('{', '[' or 0)
  auto container = [&](int L) -> uint32_t {
    if (L <= 0) return 0u;
    if (lcnt) return ((lbits >> (lcnt - 1)) & 1u) ? '[' : '{';
    if (L == ext_level) return ext_kind;
    uint32_t kind = 0;
    bool found = false;
    for (int l = before_min < L ? int(lane) - 1 : -1; l >= 0 && !found; l--) {
      if (sm.lane_min[l] >= L) continue;
      for (int j = ITEMS - 1; j >= 0; j--) {
        const uint32_t q = uint32_t(l) * ITEMS + uint32_t(j);
        if (sm.dep[q] < L) {
          kind = sm.ty[q + 2];
          found = true;
          break;
        }
      }
    }
    if (!found) {
      const uint32_t slot = uint32_t(L - 1);
      if (slot < d_in && slot < g.words * 32u) kind = ((pre[2 + (slot >> 5)] >> (slot & 31u)) & 1u) ? '[' : '{';
    }
    ext_level = L;
    ext_kind = kind;
    return kind;
  };
  auto flush = [&]() {
    if (seg_err != kNone) report(seg_pos, seg_err, seg_idx);
    seg_err = kNone;
  };
  for (int j = 0; j < ITEMS; j++) {
    const uint32_t i = i0 + j, k = tile0 + i;
    if (k >= g.n) break;
    const bool st = start_at(g.starts, k);
    if (st) {
      if (j) flush();
      lbits = 0;
      lcnt = 0;
      ext_level = -1;
    }
    const uint32_t t = sm.ty[i + 2];
    const int D = sm.dep[i];
    const int dl = delta_at(g, sm, tile0, i, h);
    if (seg_err == kNone) {
      // what the walk expects at k
      uint32_t exp;
      uint32_t p1 = st ? 0xFFu : sm.ty[i + 1];
      if (st) {
        exp = kExpRoot;
      } else if (p1 == '{') {
        exp = t == '}' ? kExpDone : kExpKey;
      } else if (p1 == '[') {
        exp = t == ']' ? kExpDone : kExpValue;
      } else if (p1 == ':') {
        exp = kExpValue;
      } else if (p1 == ',') {
        exp = container(D) == '{' ? kExpKey : kExpValue;
      } else if (p1 == '"') {
        const bool prev_start = h.start_before(g, k);
        const uint32_t p2 = prev_start ? 0xFFu : sm.ty[i];
        exp = (!prev_start && (p2 == '{' || (p2 == ',' && container(D) == '{'))) ? kExpColon : kExpAfter;
      } else {
        exp = kExpAfter;
      }
      uint32_t code = 0;
      const bool empty = is_open(t) && dl == 0;
      if (exp == kExpRoot) {
        if (g.whole && h.root_at(k) && ((t == '{' && last_type != '}') || (t == '[' && last_type != ']'))) code = kTapeError;
        else code = value_error(g, k, t, empty, D, true);
      } else if (exp == kExpValue) {
        code = value_error(g, k, t, empty, D, false);
      } else if (exp == kExpKey) {
        code = t == '"' ? 0u : ((t == 0 && (g.payload[k] & 0xFFu) == kStringError) ? kStringError : kTapeError);
      } else if (exp == kExpColon) {
        code = t == ':' ? 0u : kTapeError;
      } else if (exp == kExpAfter) {
        const uint32_t c = container(D);
        code = (c != 0 && (t == ',' || (t == '}' && c == '{') || (t == ']' && c == '['))) ? 0u : kTapeError;
      }
      if (code) {
        seg_err = code;
        seg_pos = k;
        seg_idx = k;
      }
    }
    // the lane's stack after k
    if (dl == 1) {
      if (lcnt < 32) {
        lbits = (lbits & ~(1u << lcnt)) | ((t == '[' ? 1u : 0u) << lcnt);
        lcnt++;
      }
    } else if (dl == -1 && lcnt) {
      lcnt--;
    }
    // the end of k's document: the walk must have finished its root value exactly here
    const bool last = (k + 1 == g.n || start_at(g.starts, k + 1)) && h.ends_at(g, k);
    if (last && seg_err == kNone) {
      const bool done = D + dl == 0 && (is_scalar(t) || is_close(t));
      if (!done) {
        seg_err = kTapeError;
        seg_pos = k;
        seg_idx = k + 1;
      }
    }
  }
  flush();
  sj_syncwarp();
}

// ---- one rank of a sharded pass (sjb200_document_errors_sharded): the pieces its kernels (sjb200_grammar.cu) and the
// host emulation (tests/grammar_shards_emul.cpp) share.

// the edge words of the rank (sjb200_params.h): n, ndocs, kGramEdge* flags, max_depth, the types of structurals 0, 1,
// n - 2, n - 1 (0xFF: none), the table's first entry.  first / last: the table's first and last entries (ndocs > 0).
SJ_DEV void shard_edge_words(const uint8_t *type, uint32_t n, bool whole, uint32_t ndocs, uint32_t first, uint32_t last, bool bad, bool failed,
                             uint32_t max_depth_word, uint32_t *w) {
  w[0] = n; w[1] = whole ? 0u : ndocs; w[2] = 0; w[3] = max_depth_word; w[4] = 0xFFFFFFFFu; w[5] = 0;
  if (failed) {
    w[2] = kGramEdgeFailed;
    return;
  }
  const bool table = !whole && ndocs;
  w[2] = (whole ? kGramEdgeWhole : 0u) | (bad ? kGramEdgeBadTable : 0u) | (table && first == 0 ? kGramEdgeFirstStarts : 0u) |
         (table && n && last == n - 1 ? kGramEdgeLastStarts : 0u);
  if (n) {
    const uint32_t t0 = sj_ldg_u8(type), tl = sj_ldg_u8(type + n - 1);
    const uint32_t t1 = n >= 2 ? sj_ldg_u8(type + 1) : 0xFFu, tm = n >= 2 ? sj_ldg_u8(type + n - 2) : 0xFFu;
    w[4] = t0 | (t1 << 8) | (tm << 16) | (tl << 24);
  }
  w[5] = table ? first : 0u;
}

// The stack entering rank `rank`: the records of ranks 0 .. rank - 1 folded in order into dst (2 + words words).  rec(r,
// k) is word k of rank r's record; acc and child are the warp's shared scratch.
template <class W>
SJ_DEV void shard_incoming(unsigned lane, uint32_t *acc, uint32_t *child, W &&rec, uint32_t rank, uint32_t words, uint32_t *dst) {
  if (lane < 2) acc[lane] = 0;
  sj_syncwarp();
  for (uint32_t r = 0; r < rank; r++) {
    for (uint32_t k = lane; k < 2 + words; k += 32) child[k] = rec(r, k);
    sj_syncwarp();
    compose(lane, acc, child, words);
  }
  copy_record(lane, dst, acc);
}

// the slot of first[] that an error of document d (kNone: before the rank's first document start) goes to: the document,
// or the leading segment's slot `owned`.  Whole mode: slot 0 is rank 0's document, or the leading segment elsewhere.
SJ_DEV uint32_t shard_slot(bool whole, uint32_t d, uint32_t owned) { return whole ? 0u : (d == kNone ? owned : d); }

// the result of a document that starts on the rank and ends on it: its first error (key = index << 8 | code, local), or
// SUCCESS one past its value (next: the local start of the next document)
SJ_DEV void shard_doc_result(unsigned long long key, uint64_t tokens_before, uint32_t next, int32_t *error, uint64_t *index) {
  if (key != ~0ull) {
    *error = int32_t(key & 0xFFu);
    *index = tokens_before + (key >> 8);
  } else {
    *error = 0;
    *index = tokens_before + next;
  }
}

SJ_DEV unsigned long long shard_global_key(unsigned long long key, uint64_t tokens_before) {
  return key == ~0ull ? key : key + (static_cast<unsigned long long>(tokens_before) << 8);
}

// the result words of the rank (sjb200_params.h): its leading segment's first error, its last document's (global keys),
// its other documents in error and the first of them (first_doc, kNone: none) with its key
SJ_DEV void shard_result_words(const unsigned long long *first, uint32_t owned, uint64_t tokens_before, uint32_t errors, uint32_t first_doc, uint32_t *w) {
  const unsigned long long lead = shard_global_key(first[owned], tokens_before), last = owned ? shard_global_key(first[owned - 1], tokens_before) : ~0ull;
  const unsigned long long fk = first_doc != kNone ? shard_global_key(first[first_doc], tokens_before) : ~0ull;
  w[0] = uint32_t(lead); w[1] = uint32_t(lead >> 32); w[2] = uint32_t(last); w[3] = uint32_t(last >> 32);
  w[4] = errors; w[5] = first_doc; w[6] = uint32_t(fk); w[7] = uint32_t(fk >> 32);
}

}  // namespace gram
}  // namespace sjb200
