// sjb200_column.cuh -- typed columns from JSON Pointer results (sjb200_column_dev): the row rules of the DOM getters
// (element::get_int64 / get_uint64 / get_bool / get_string, get_array().size(), get_object().size()) over the
// stage-2-lite tokens, the container size walk and the string copy, written against sjb200_simt.cuh so that the host
// SIMT emulation (tests/column_emul.cpp) runs the same source as the sm_90a kernels in sjb200_column.cu.
//
// A row is one sjb200_at_pointer_dev result {error, structural index}.  Its value follows from the tokens alone: the
// type char, the integer payload, the string record [u32 length][bytes][0] in the string buffer, and for a container
// the structurals up to its close.  The size walk is find_child's (sjb200_pointer.cuh) without a target: the group
// prefix sum of bracket deltas gives each structural's depth relative to the container, and the children are counted
// at depth 0 up to the first close there.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "sjb200_pointer.cuh"

namespace sjb200 {
namespace col {

using ptr::kIncorrectType;
using ptr::kNone;
using ptr::kUnexpectedError;
constexpr int32_t kNumberOutOfRange = 18;  // simdjson::NUMBER_OUT_OF_RANGE
constexpr uint32_t kCountSat = 0xFFFFFF;   // tape_builder::end_container's cntsat (src/generic/stage2/tape_builder.h L411)

enum Kind { kInt64 = 1, kUint64 = 2, kBool = 3, kString = 4, kArraySize = 5, kObjectSize = 6 };  // SJB200_COLUMN_*

struct Row {  // sjb200_pointer_result
  int32_t error;
  uint32_t index;
};

struct Cols {
  const uint8_t *type;      // sjb200_tokens_dev d_type
  const uint64_t *payload;  // ... d_payload
  uint32_t n;
  const uint8_t *strbuf;    // ... d_strbuf, string_bytes in use
  uint64_t string_bytes;
  const Row *rows;
  uint32_t nrows;
};

SJ_DEV bool is_value(uint32_t t) {
  return t == '{' || t == '[' || t == '"' || t == 'l' || t == 'u' || t == 'd' || t == 't' || t == 'f' || t == 'n';
}

// What row r selects: err != 0 (a row in error keeps its error; an index past n or at a token that is not a value is
// UNEXPECTED_ERROR), else the structural k and its type.
struct Pick {
  int32_t err;
  uint32_t type;
  uint32_t k;
};
SJ_DEV Pick pick_row(const Cols &c, uint32_t r) {
  const Row row = c.rows[r];
  if (row.error != 0) return Pick{row.error, 0, 0};
  if (row.index >= c.n) return Pick{kUnexpectedError, 0, 0};
  const uint32_t t = c.type[row.index];
  if (!is_value(t)) return Pick{kUnexpectedError, 0, 0};
  return Pick{0, t, row.index};
}

// The bytes of the string at structural k: [*off, *off + *len) of the string buffer.  false: its record (length word,
// bytes and terminator) does not lie inside [0, string_bytes); nothing outside is read.
SJ_DEV bool string_record(const Cols &c, uint32_t k, uint64_t *off, uint32_t *len) {
  const uint64_t o = c.payload[k];
  if (o > c.string_bytes || c.string_bytes - o < 5) return false;
  const uint8_t *p = c.strbuf + o;
  const uint32_t l = uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24);
  if (c.string_bytes - o - 5 < l) return false;
  *off = o + 4;
  *len = l;
  return true;
}

// The getter of a scalar kind on a value of type t with payload v: the error, *out the value (0 on an error)
// (include/simdjson/dom/element-inl.h: get_int64 L280-294, get_uint64 L266-279, get_bool)
SJ_DEV int32_t scalar_rule(int kind, uint32_t t, uint64_t v, uint64_t *out) {
  *out = 0;
  if (kind == kInt64) {
    if (t != 'l' && t != 'u') return kIncorrectType;
    if (t == 'u' && v > uint64_t(INT64_MAX)) return kNumberOutOfRange;
    *out = v;
    return 0;
  }
  if (kind == kUint64) {
    if (t != 'l' && t != 'u') return kIncorrectType;
    if (t == 'l' && int64_t(v) < 0) return kNumberOutOfRange;
    *out = v;
    return 0;
  }
  if (t != 't' && t != 'f') return kIncorrectType;  // kBool
  *out = t == 't' ? 1 : 0;
  return 0;
}

// ---- the size walk
// Where a count stands: the next structural to read, the depth relative to the container entering it, the children so far.
struct SizeAt {
  uint32_t pos;
  int32_t depth;
  uint32_t count;
};

// The children of an array (obj = false: the structurals at relative depth 0 other than ',') or of an object (obj =
// true: the strings at depth 0 followed by ':') from *at on, by group g, reading at most `limit` structurals from
// at->pos and none at or past n.  true: the container's close at depth 0, or n, was reached and at->count is the
// count (unsaturated); false: *at is where to go on.
template <class G, int ITEMS>
SJ_DEV bool count_children(G &g, const uint8_t *type, uint32_t n, bool obj, SizeAt *at, uint64_t limit) {
  uint64_t pos = at->pos;
  int depth = at->depth;
  uint32_t count = at->count;
  const uint64_t stop = limit >> 32 ? ~0ull : pos + limit;  // (pos < 2^32)
  for (;; pos += uint64_t(G::kWidth) * ITEMS) {
    if (pos >= n) break;
    if (pos >= stop) {
      *at = SizeAt{uint32_t(pos), depth, count};
      return false;
    }
    const uint64_t k0 = pos + uint64_t(g.rank()) * ITEMS;
    uint32_t t[ITEMS];
    int sum = 0;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
      t[i] = k0 + i < n ? uint32_t(type[k0 + i]) : 0u;
      sum += ptr::tok_delta(t[i]);
    }
    int total_delta;
    const int d_in = depth + g.scan(sum, &total_delta);
    uint32_t close_at = kNone;
    int d = d_in;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
      if (d == 0 && close_at == kNone && ptr::tok_close(t[i])) close_at = uint32_t(k0 + i);
      d += ptr::tok_delta(t[i]);
    }
    const uint32_t first_close = g.min(close_at);
    int kids = 0;
    d = d_in;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
      const uint64_t k = k0 + i;
      if (d == 0 && k < n && k < first_close && !ptr::tok_close(t[i]))
        kids += obj ? (t[i] == '"' && k + 1 < n && type[k + 1] == ':') : (t[i] != ',');
      d += ptr::tok_delta(t[i]);
    }
    int total_kids;
    g.scan(kids, &total_kids);
    count += uint32_t(total_kids);
    if (first_close != kNone) break;
    depth += total_delta;
  }
  *at = SizeAt{uint32_t(pos < n ? pos : n), depth, count};
  return true;
}

// ---- the string copy
// len bytes from src to dst by the `width` threads of a group, this one being `rank`.  The destination leaves in aligned
// 16-byte vectors (the bytes before the first and after the last one singly); a vector is assembled from the two
// aligned source vectors it straddles when both lie inside [src, src + len), else byte by byte.  Nothing outside
// [src, src + len) is read, nothing outside [dst, dst + len) written.
SJ_DEV void group_copy(unsigned rank, unsigned width, uint8_t *dst, const uint8_t *src, uint64_t len) {
  const uint64_t to_al = (16u - (uintptr_t(dst) & 15u)) & 15u;
  const uint64_t head = len < to_al ? len : to_al;
  const uint64_t nvec = (len - head) >> 4;
  const uint64_t tail = head + (nvec << 4);
  for (uint64_t i = rank; i < head; i += width) dst[i] = src[i];
  for (uint64_t i = tail + rank; i < len; i += width) dst[i] = src[i];
  const uint8_t *s = src + head;
  const uint32_t sh = uint32_t(uintptr_t(s) & 15u);
  const uint8_t *s_al = s - sh;
  sj_u4 *dv = reinterpret_cast<sj_u4 *>(dst + head);
  for (uint64_t v = rank; v < nvec; v += width) {
    const uint8_t *a = s_al + 16 * v;  // the aligned source vector holding the vector's first byte
    uint32_t o[4];
    if (sh == 0) {
      const sj_u4 x = sj_ldg_u4(a);
      o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w;
    } else if (a >= src && a + 32 <= src + len) {
      const sj_u4 x = sj_ldg_u4(a), y = sj_ldg_u4(a + 16);
      const uint32_t w[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
      const uint32_t q = sh >> 2;
      const int r = int(sh & 3u) * 8;
      uint32_t p[5];
#pragma unroll
      for (int j = 0; j < 5; j++) p[j] = q == 0 ? w[j] : (q == 1 ? w[j + 1] : (q == 2 ? w[j + 2] : w[j + 3]));
#pragma unroll
      for (int j = 0; j < 4; j++) o[j] = sj_funnel_r(p[j], p[j + 1], r);
    } else {
      const uint8_t *b = s + 16 * v;
#pragma unroll
      for (int j = 0; j < 4; j++)
        o[j] = uint32_t(b[4 * j]) | (uint32_t(b[4 * j + 1]) << 8) | (uint32_t(b[4 * j + 2]) << 16) | (uint32_t(b[4 * j + 3]) << 24);
    }
    dv[v] = sj_make_u4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace col
}  // namespace sjb200
