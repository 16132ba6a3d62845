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

// The children of the container whose opening structural is c, searched for the key (object) or index (array) of level
// l.  Returns the structural index of the selected value, or kNone with *err set.  Structurals at or past `end` are never
// read; a container that is not closed before it (a document the reference rejects for its nesting) ends the search.
template <class G, int ITEMS>
SJ_DEV uint32_t find_child(G &g, const Walk &w, uint32_t c, bool obj, const PtrLevel &l, uint32_t end, int32_t *err) {
  int depth = 0;        // relative depth entering this step
  uint32_t ord = 0;     // array elements before this step
  for (uint64_t pos = uint64_t(c) + 1;; pos += uint64_t(G::kWidth) * ITEMS) {
    if (pos >= end) break;
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
          if (hit == kNone && close_at == kNone && t[i] == '"' && k + 2 < end && w.type[k + 1] == ':' && key_equals(w, w.payload[k], l))
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

// One (document, pointer) pair: from the document's root structural, every level of the pointer.  Returns the selected
// structural index or kNone with *err set.
template <class G, int ITEMS>
SJ_DEV uint32_t walk_pointer(G &g, const Walk &w, const PtrHeader &h, uint32_t root, uint32_t end, int32_t *err) {
  *err = 0;
  if (h.error != 0) {
    *err = h.error;
    return kNone;
  }
  uint32_t v = root;
  for (uint32_t L = 0; L < h.nlevels; L++) {
    const PtrLevel l = w.levels[h.level0 + L];
    const uint32_t t = w.type[v];
    const bool obj = t == '{';
    if (!obj && t != '[') {
      *err = l.scalar_error;
      return kNone;
    }
    if (obj ? l.key_error != 0 : l.array_error != 0) {
      *err = obj ? l.key_error : l.array_error;
      return kNone;
    }
    int32_t e = 0;
    v = find_child<G, ITEMS>(g, w, v, obj, l, end, &e);
    if (v == kNone || v >= end) {
      *err = e ? e : (obj ? kNoSuchField : kIndexOutOfBounds);
      return kNone;
    }
  }
  return v;
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
