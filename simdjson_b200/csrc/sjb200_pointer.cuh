// sjb200_pointer.cuh -- JSON Pointer lookup over the stage-2-lite tokens (sjb200_at_pointer_dev): the structural walk of
// one (document, pointer) pair by a group of threads, written against sjb200_simt.cuh so that the host SIMT emulation
// (tests/pointer_emul.cpp) runs the same source as the sm_90a kernels in sjb200_pointer.cu.
//
// The pointer's string grammar is decided on the host (compile_pointers): each reference token becomes one PtrLevel,
// and the walk only follows structure.  It needs no depth array and no tape: a group starts at a container and scans
// forward, G * ITEMS structurals per step; the depth relative to the container is a group prefix sum of +1 for '{' '['
// and -1 for '}' ']'; the container's children are the structurals at relative depth 0 and the first close at depth 0
// ends it.  The lowest match wins (the first key in document order), and the next level starts right after the value it
// selects, so no structural is read twice.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "sjb200_simt.cuh"

namespace sjb200 {
namespace ptr {

// simdjson::error_code values of the lookup (include/simdjson/error.h L19-54)
constexpr int32_t kIncorrectType = 17, kIndexOutOfBounds = 19, kNoSuchField = 20, kInvalidJsonPointer = 22, kUnexpectedError = 24;
constexpr uint32_t kNone = 0xFFFFFFFFu;

struct PtrHeader {
  uint32_t level0;    // first PtrLevel of this pointer
  uint32_t nlevels;   // reference tokens; 0 with error 0: the root
  int32_t error;      // != 0: the pointer fails before any token (a non-empty pointer without a leading '/')
  uint32_t reserved;
};
struct PtrLevel {
  uint32_t key_off;     // the unescaped key, bytes [key_off, key_off + key_len) of the key blob
  uint32_t key_len;
  int32_t key_error;    // at an object: INVALID_JSON_POINTER for a '~' escape other than ~0 / ~1, else 0
  int32_t array_error;  // at an array: 0, or the error of the token as an index (incl. a last token "-")
  uint32_t array_index; // at an array, array_error == 0: the index (>= 2^32 - 1 folds into INDEX_OUT_OF_BOUNDS)
  int32_t scalar_error; // at a scalar: NO_SUCH_FIELD when the remainder from this token is well formed, else INVALID
};

struct Walk {
  const uint8_t *type;      // sjb200_tokens_dev d_type
  const uint64_t *payload;  // ... d_payload
  const uint8_t *strbuf;    // ... d_strbuf
  uint64_t string_bytes;
  const PtrLevel *levels;
  const uint8_t *keys;
};

SJ_DEV int tok_delta(uint32_t t) { return (t == '{' || t == '[') ? 1 : ((t == '}' || t == ']') ? -1 : 0); }
SJ_DEV bool tok_close(uint32_t t) { return t == '}' || t == ']'; }

// the string record at payload offset `off` ([u32 length][bytes][0]) equals the key; never reads past string_bytes
SJ_DEV bool key_equals(const Walk &w, uint64_t off, const PtrLevel &l) {
  if (off + 4 > w.string_bytes) return false;
  const uint8_t *r = w.strbuf + off;
  const uint32_t len = uint32_t(r[0]) | (uint32_t(r[1]) << 8) | (uint32_t(r[2]) << 16) | (uint32_t(r[3]) << 24);
  if (len != l.key_len || off + 4 + len > w.string_bytes) return false;
  for (uint32_t i = 0; i < len; i++)
    if (r[4 + i] != w.keys[l.key_off + i]) return false;
  return true;
}

// A warp as the group: one structural per lane per step.
struct WarpGroup {
  static constexpr unsigned kWidth = 32;
  unsigned lane;
  SJ_DEV unsigned rank() const { return lane; }
  // exclusive prefix sum over the group; *total = the sum of all
  SJ_DEV int scan(int x, int *total) const {
    int v = x;
    for (int d = 1; d < 32; d <<= 1) {
      const int u = int(sj_shfl_up(uint32_t(v), d));
      if (int(lane) >= d) v += u;
    }
    *total = int(sj_shfl(uint32_t(v), 31));
    return v - x;
  }
  SJ_DEV uint32_t min(uint32_t x) const { return sj_reduce_min(x); }
};

// A CTA of W warps as the group.  Shared scratch: two alternating halves, so one barrier per collective suffices (a
// thread can be at most one collective ahead of the slowest, and that one reads the other half).
template <unsigned W>
struct CtaSmem {
  int32_t part[2][W];
};
template <unsigned W>
struct CtaGroup {
  static constexpr unsigned kWidth = 32 * W;
  unsigned tid;
  CtaSmem<W> *sm;
  unsigned phase = 0;
  SJ_DEV unsigned rank() const { return tid; }
  SJ_DEV int scan(int x, int *total) {
    const unsigned lane = tid & 31u, warp = tid >> 5;
    int v = x;
    for (int d = 1; d < 32; d <<= 1) {
      const int u = int(sj_shfl_up(uint32_t(v), d));
      if (int(lane) >= d) v += u;
    }
    if (lane == 31) sm->part[phase][warp] = v;
    sj_syncthreads();
    int before = 0, all = 0;
    for (unsigned k = 0; k < W; k++) {
      const int p = sm->part[phase][k];
      before += k < warp ? p : 0;
      all += p;
    }
    phase ^= 1u;
    *total = all;
    return before + v - x;
  }
  SJ_DEV uint32_t min(uint32_t x) {
    const uint32_t m = sj_reduce_min(x);
    if ((tid & 31u) == 0) sm->part[phase][tid >> 5] = int32_t(m);
    sj_syncthreads();
    uint32_t r = kNone;
    for (unsigned k = 0; k < W; k++) r = uint32_t(sm->part[phase][k]) < r ? uint32_t(sm->part[phase][k]) : r;
    phase ^= 1u;
    return r;
  }
};

// Where a cut between ranks stops a walk (sjb200_at_pointer_sharded).  NoCut: the unsharded walk, every structural of
// the document lies in [0, end).  ShardCut: one rank's piece of a document whose structurals go on past this rank's
// last one when `continues`; the walk then reads nothing at or past `end` (the rank's n), takes the type of the
// structural after it from the halo, and suspends where the unsharded walk would run into the end.
struct NoCut {
  static constexpr bool kSuspends = false;
  static constexpr uint32_t continues = 0;
  // is the key string at k followed by its ':' and a value inside the document
  SJ_DEV bool key_at(const Walk &w, uint64_t k, uint32_t end) const { return k + 2 < end && w.type[k + 1] == ':'; }
};
struct ShardCut {
  static constexpr bool kSuspends = true;
  uint32_t next_type;  // type of the structural after this rank's last one (the next holder's structural 0)
  uint32_t continues;  // the document goes on past this rank's last structural
  uint64_t doc_end;    // the document's end, counted from this rank's structural 0 (end itself when !continues)
  SJ_DEV bool key_at(const Walk &w, uint64_t k, uint32_t end) const {
    return k + 2 < doc_end && (k + 1 < end ? uint32_t(w.type[k + 1]) : next_type) == ':';
  }
};
constexpr uint32_t kSuspend = 0xFFFFFFFEu;  // find_child / walk_from: the walk reached the end of a piece inside its document

// a search inside a container: the relative depth and the array elements counted before the next structural
struct Cursor {
  int32_t depth;
  uint32_t ord;
};

// The children of a container, from structural pos on (its opener + 1, or where a suspended search resumes with *cur),
// searched for the key (object) or index (array) of level l.  Returns the structural index of the selected value
// (with a ShardCut possibly past end: a key whose ':' or value lies across the cut), kNone with *err set, or kSuspend
// with *cur at end.  Structurals at or past `end` are never read; a container that is not closed before it (a document
// the reference rejects for its nesting) ends the search.
template <class G, int ITEMS, class C>
SJ_DEV uint32_t find_child(G &g, const Walk &w, uint64_t pos, bool obj, const PtrLevel &l, uint32_t end, const C &cut, Cursor *cur, int32_t *err) {
  int depth = cur->depth;  // relative depth entering this step
  uint32_t ord = cur->ord;  // array elements before this step
  for (;; pos += uint64_t(G::kWidth) * ITEMS) {
    if (pos >= end) {
      if (C::kSuspends && cut.continues) {
        *cur = Cursor{depth, ord};
        return kSuspend;
      }
      break;
    }
    const uint64_t k0 = pos + uint64_t(g.rank()) * ITEMS;
    uint32_t t[ITEMS];
    int sum = 0;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
      t[i] = k0 + i < end ? uint32_t(w.type[k0 + i]) : 0u;
      sum += tok_delta(t[i]);
    }
    int total_delta;
    const int d_in = depth + g.scan(sum, &total_delta);
    // first pass over the items: the first close at depth 0, the first matching key (object) / the element count (array)
    uint32_t close_at = kNone, hit = kNone, elems = 0;
    int d = d_in;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
      const uint64_t k = k0 + i;
      if (d == 0 && k < end) {
        if (tok_close(t[i])) {
          if (close_at == kNone) close_at = uint32_t(k);
        } else if (obj) {
          if (hit == kNone && close_at == kNone && t[i] == '"' && cut.key_at(w, k, end) && key_equals(w, w.payload[k], l))
            hit = uint32_t(k);
        } else if (t[i] != ',' && close_at == kNone) {
          elems++;
        }
      }
      d += tok_delta(t[i]);
    }
    uint32_t total_elems = 0;
    if (!obj) {
      int te;
      uint32_t before = ord + uint32_t(g.scan(int(elems), &te));
      total_elems = uint32_t(te);
      // second pass: the element whose ordinal is the index
      d = d_in;
#pragma unroll
      for (int i = 0; i < ITEMS; i++) {
        const uint64_t k = k0 + i;
        if (d == 0 && k < end && uint32_t(k) < close_at && !tok_close(t[i]) && t[i] != ',') {
          if (before == l.array_index && hit == kNone) hit = uint32_t(k);
          before++;
        }
        d += tok_delta(t[i]);
      }
    }
    const uint32_t first_close = g.min(close_at);
    const uint32_t first_hit = g.min(hit);
    if (first_hit != kNone && (first_close == kNone || first_hit < first_close)) {
      if (!obj) return first_hit;
      *err = 0;
      return first_hit + 2;  // key ':' value
    }
    if (first_close != kNone) break;
    depth += total_delta;
    ord += total_elems;
  }
  *err = obj ? kNoSuchField : kIndexOutOfBounds;
  return kNone;
}

// Where a walk of one pointer stands: about to take reference token `level` at the value `pos` (open = 0), or inside
// that token's container (open = 1, its kind in obj), searching on from structural pos with the relative depth and the
// array elements counted so far.  A suspended walk's state, relative to the start of the next piece.
struct WalkAt {
  uint32_t level;
  uint32_t pos;
  int32_t depth;
  uint32_t ord;
  uint32_t open;
  uint32_t obj;
};

// One (document, pointer) pair from `at` on, every remaining level of the pointer.  Returns the selected structural
// index, kNone with *err set, or (ShardCut only) kSuspend with *susp: where the walk goes on at the next piece.  With a
// ShardCut the selected index may lie past end (the value of a key on this rank).
template <class G, int ITEMS, class C>
SJ_DEV uint32_t walk_from(G &g, const Walk &w, const PtrHeader &h, WalkAt at, uint32_t end, const C &cut, int32_t *err, WalkAt *susp) {
  *err = 0;
  if (h.error != 0) {
    *err = h.error;
    return kNone;
  }
  uint32_t v = at.pos;
  for (uint32_t L = at.level; L < h.nlevels; L++) {
    const PtrLevel l = w.levels[h.level0 + L];
    bool obj;
    uint64_t pos;
    Cursor cur{0, 0};
    if (C::kSuspends && at.open) {
      at.open = 0;
      obj = at.obj != 0;
      pos = v;
      cur = Cursor{at.depth, at.ord};
    } else {
      if (C::kSuspends && v >= end) {  // the value of this level lies on a later rank
        *susp = WalkAt{L, v - end, 0, 0, 0, 0};
        return kSuspend;
      }
      const uint32_t t = w.type[v];
      obj = t == '{';
      if (!obj && t != '[') {
        *err = l.scalar_error;
        return kNone;
      }
      if (obj ? l.key_error != 0 : l.array_error != 0) {
        *err = obj ? l.key_error : l.array_error;
        return kNone;
      }
      pos = uint64_t(v) + 1;
    }
    int32_t e = 0;
    v = find_child<G, ITEMS>(g, w, pos, obj, l, end, cut, &cur, &e);
    if (C::kSuspends && v == kSuspend) {
      *susp = WalkAt{L, 0, cur.depth, cur.ord, 1, obj ? 1u : 0u};
      return kSuspend;
    }
    if (v == kNone || (!C::kSuspends && v >= end)) {
      *err = e ? e : (obj ? kNoSuchField : kIndexOutOfBounds);
      return kNone;
    }
  }
  return v;
}

// One (document, pointer) pair: from the document's root structural, every level of the pointer.  Returns the selected
// structural index or kNone with *err set.
template <class G, int ITEMS>
SJ_DEV uint32_t walk_pointer(G &g, const Walk &w, const PtrHeader &h, uint32_t root, uint32_t end, int32_t *err) {
  WalkAt susp;
  return walk_from<G, ITEMS>(g, w, h, WalkAt{0, root, 0, 0, 0, 0}, end, NoCut{}, err, &susp);
}

// One rank's view of the document that holds its last structural (sjb200_at_pointer_sharded; sjb200_pointer_edge_fold).
struct ShardView {
  uint32_t n;               // this rank's structurals
  uint32_t next_type;       // type of the structural after its last one (0xFF: none)
  uint32_t tail_continues;  // the document holding structural n - 1 goes on past this rank
  uint64_t tail_end;        // n + that document's structurals on later ranks
};
// the cut of a piece [.., end) of this rank's structurals: a piece that ends at n belongs to the document holding n - 1
SJ_DEV ShardCut piece_cut(const ShardView &v, uint32_t end) {
  const bool c = v.tail_continues != 0 && end == v.n;
  return ShardCut{v.next_type, c ? 1u : 0u, c ? v.tail_end : uint64_t(end)};
}

// A suspended walk as the 16-byte record a rank hands to the next holder of its document (sjb200_at_pointer_sharded):
//   w0 = seq << 32 | step << 24 | obj << 18 | open << 17 | pos << 16 | level     w1 = ord << 32 | depth
// pos is 0 or 1 (a value right after the cut, or after its ':'); step tells the double-buffered rounds apart.
SJ_DEV void pack_walk(const WalkAt &a, uint32_t seq, uint32_t step, unsigned long long *w0, unsigned long long *w1) {
  *w0 = (static_cast<unsigned long long>(seq) << 32) | (static_cast<unsigned long long>(step & 0xFFu) << 24) |
        (static_cast<unsigned long long>(a.obj & 1u) << 18) | (static_cast<unsigned long long>(a.open & 1u) << 17) |
        (static_cast<unsigned long long>(a.pos & 1u) << 16) | (a.level & 0xFFFFu);
  *w1 = (static_cast<unsigned long long>(a.ord) << 32) | uint32_t(a.depth);
}
// false: the record is not of (seq, step) -- no walk of this pointer was handed over in that step
SJ_DEV bool unpack_walk(unsigned long long w0, unsigned long long w1, uint32_t seq, uint32_t step, WalkAt *a) {
  if (uint32_t(w0 >> 32) != seq || uint32_t(w0 >> 24 & 0xFFu) != (step & 0xFFu)) return false;
  *a = WalkAt{uint32_t(w0 & 0xFFFFu), uint32_t(w0 >> 16) & 1u, int32_t(uint32_t(w1)), uint32_t(w1 >> 32), uint32_t(w0 >> 17) & 1u, uint32_t(w0 >> 18) & 1u};
  return true;
}

// ---- host: the pointers of one call compiled into one blob [PtrHeader x np][PtrLevel x levels][key bytes], so that
// all of the pointer's string grammar (element::at_pointer, object / array::at_pointer, parse_json_pointer_array_index)
// is decided here once and the device only follows structure.
constexpr int kMaxPointers = 65536;        // SJB200_POINTER_MAX_POINTERS
constexpr uint32_t kMaxTokens = 1024;      // SJB200_POINTER_MAX_TOKENS
constexpr size_t kMaxPointerBytes = 1u << 20;  // SJB200_POINTER_MAX_BYTES

struct CompiledPointers {
  std::vector<PtrHeader> headers;
  std::vector<PtrLevel> levels;
  std::string keys;
};

// is_pointer_well_formed (include/simdjson/dom/element-inl.h L410-425): only the first '~' is looked at
inline bool pointer_well_formed(const char *p, size_t len) {
  if (len == 0 || p[0] != '/') return false;
  for (size_t i = 0; i < len; i++)
    if (p[i] == '~') return i + 1 < len && (p[i + 1] == '0' || p[i + 1] == '1');
  return true;
}

// 0 (SUCCESS), 1 (CAPACITY: a limit above) or 24 (UNEXPECTED_ERROR: a null pointer with a non-zero length)
inline int compile_pointers(const char *const *ptrs, const size_t *lens, int np, CompiledPointers *out) {
  out->headers.assign(size_t(np > 0 ? np : 0), PtrHeader{0, 0, 0, 0});
  out->levels.clear();
  out->keys.clear();
  if (np > kMaxPointers) return 1;
  size_t bytes = 0;
  for (int p = 0; p < np; p++) {
    const char *s = ptrs[p];
    const size_t len = lens[p];
    if (len && !s) return 24;
    if ((bytes += len) > kMaxPointerBytes) return 1;
    PtrHeader &h = out->headers[size_t(p)];
    h.level0 = uint32_t(out->levels.size());
    if (len == 0) continue;  // "": the root
    if (s[0] != '/') {
      h.error = kInvalidJsonPointer;
      continue;
    }
    for (size_t at = 0; at < len;) {  // s[at] == '/': one reference token up to the next '/'
      size_t e = at + 1;
      while (e < len && s[e] != '/') e++;
      if (++h.nlevels > kMaxTokens) return 1;
      PtrLevel l{uint32_t(out->keys.size()), 0, 0, 0, 0, 0};
      const char *t = s + at + 1;
      const size_t tl = e - at - 1;
      // object: ~0 -> '~', ~1 -> '/', any other '~' is INVALID_JSON_POINTER (object-inl.h L115-134)
      for (size_t i = 0; i < tl; i++) {
        if (t[i] != '~') {
          out->keys.push_back(t[i]);
        } else if (i + 1 < tl && (t[i + 1] == '0' || t[i + 1] == '1')) {
          out->keys.push_back(t[i + 1] == '0' ? '~' : '/');
          i++;
        } else {
          l.key_error = kInvalidJsonPointer;
          break;
        }
      }
      l.key_len = uint32_t(out->keys.size() - l.key_off);
      // array: a last token "-" is past the end (array-inl.h L107), else parse_json_pointer_array_index (jsonpathutil.h)
      if (e == len && tl == 1 && t[0] == '-') {
        l.array_error = kIndexOutOfBounds;
      } else {
        uint64_t v = 0;
        size_t i = 0;
        for (; i < tl; i++) {
          const uint8_t digit = uint8_t(t[i] - '0');
          if (digit > 9) { l.array_error = kIncorrectType; break; }
          if (i > 0 && t[0] == '0') { l.array_error = kInvalidJsonPointer; break; }
          if (v > (UINT64_MAX - digit) / 10) { l.array_error = kIndexOutOfBounds; break; }
          v = v * 10 + digit;
        }
        if (l.array_error == 0 && tl == 0) l.array_error = kInvalidJsonPointer;
        if (l.array_error == 0 && v >= kNone) l.array_error = kIndexOutOfBounds;  // no array has that many elements
        l.array_index = l.array_error == 0 ? uint32_t(v) : 0;
      }
      // a scalar reached with this token and the rest still to go (element-inl.h L436-441)
      l.scalar_error = pointer_well_formed(s + at, len - at) ? kNoSuchField : kInvalidJsonPointer;
      out->levels.push_back(l);
      at = e;
    }
  }
  return 0;
}

}  // namespace ptr
}  // namespace sjb200
