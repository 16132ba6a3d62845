// sjb200_column.cu -- typed columns from JSON Pointer results on the device (sjb200_column_dev): the row rules, the size
// walk and the string copy of sjb200_column.cuh as sm_90a kernels.
//
//   scalars (INT64, UINT64, BOOL)   col_scalar_kernel: one grid-stride pass, one thread per row
//   sizes (ARRAY_SIZE, OBJECT_SIZE) col_size_warp_kernel: one warp per row, up to kCtaMinStructurals structurals; a row
//                                   still open after them is listed with its cursor and col_size_cta_kernel finishes it,
//                                   one CTA per row (the split of the pointer walks, sjb200_pointer.cu)
//   STRING                          col_string_len_kernel: the row checks and lengths, per-tile sums of the bytes and of
//                                   the rows in error; tile_scan_kernel (sjb200_tape.cu); col_string_copy_kernel: the
//                                   offsets and the copy; col_string_long_kernel: the strings over kWarpBytes, listed
//                                   chunk by chunk, one CTA per chunk
#include "sjb200_column.h"

#include "sjb200_pointer.h"
#include "sjb200_tape.h"

namespace sjb200 {
namespace col {
namespace {

constexpr int kTile = 256;                // rows per tile of the string kernels, one per thread
constexpr uint32_t kLaneBytes = 32;       // a lane copies a string of at most this many bytes itself
constexpr uint64_t kWarpBytes = 4096;     // a warp copies one of at most this many; longer ones go to col_string_long_kernel
constexpr uint32_t kOutBytes = 12 * 1024; // a tile's bytes composed in shared memory when they fit
constexpr uint64_t kChunk = 16 * 1024;    // the piece of a long string one CTA copies

struct Scratch {  // column_scratch_bytes(nrows) bytes, the layout of launch_column
  TokenTotals *tot;          // n_strings: the rows in error; string_bytes: the STRING column's bytes
  uint32_t *list_count;      // entries listed for the CTA size walk / the long-string copy
  unsigned long long *tile_sums;
  uint32_t *tile_errs;
  SizeAt *handed;            // [nrows]: a size walk handed to a CTA, .pos / .depth / .count, and the row in list_rows
  uint32_t *list_rows;       // [nrows]
  unsigned long long *chunks;  // [long_chunk_capacity(bytes_capacity)]: row << 32 | chunk of a long string
};

// A string over kWarpBytes has at most len / kWarpBytes chunks of kChunk bytes (kChunk = 4 kWarpBytes), so a column
// that fits bytes_capacity lists at most bytes_capacity / kWarpBytes of them.
size_t long_chunk_capacity(uint64_t bytes_capacity) { return size_t(bytes_capacity / kWarpBytes) + 1; }

struct Out {
  int32_t *err;
  uint8_t *row_type;
  void *values;
  int64_t *offsets;
  uint8_t *bytes;
  uint64_t capacity;
};

__device__ __forceinline__ void add_errors(TokenTotals *tot, uint32_t mine) {
  const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, mine);
  if ((threadIdx.x & 31u) == 0 && w) atomicAdd(&tot->n_strings, w);
}

// ---- scalars
__global__ void __launch_bounds__(256) col_scalar_kernel(Cols c, int kind, Out o, Scratch s) {
  uint32_t errs = 0;
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t r = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; r < c.nrows; r += stride) {
    const Pick p = pick_row(c, uint32_t(r));
    int32_t e = p.err;
    uint64_t v = 0;
    if (e == 0) e = scalar_rule(kind, p.type, c.payload[p.k], &v);
    o.err[r] = e;
    o.row_type[r] = uint8_t(p.type);
    if (kind == kBool)
      static_cast<uint8_t *>(o.values)[r] = uint8_t(v);
    else
      static_cast<uint64_t *>(o.values)[r] = v;
    errs += e != 0;
  }
  add_errors(s.tot, errs);
}

// ---- sizes
__global__ void __launch_bounds__(256) col_size_warp_kernel(Cols c, int kind, Out o, Scratch s) {
  const bool obj = kind == kObjectSize;
  const uint32_t want = obj ? '{' : '[';
  ptr::WarpGroup g{threadIdx.x & 31u};
  uint32_t errs = 0;
  const uint64_t stride = (uint64_t(gridDim.x) * blockDim.x) >> 5;
  for (uint64_t r = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; r < c.nrows; r += stride) {
    const Pick p = pick_row(c, uint32_t(r));
    int32_t e = p.err;
    uint64_t v = 0;
    if (e == 0 && p.type != want) e = kIncorrectType;
    if (e == 0) {
      SizeAt at{p.k + 1, 0, 0};
      if (!count_children<ptr::WarpGroup, 1>(g, c.type, c.n, obj, &at, ptr::kCtaMinStructurals)) {
        if (g.lane == 0) {
          const uint32_t slot = atomicAdd(s.list_count, 1u);
          s.handed[slot] = at;
          s.list_rows[slot] = uint32_t(r);
        }
        continue;  // written by col_size_cta_kernel
      }
      v = at.count < kCountSat ? at.count : kCountSat;
    }
    if (g.lane == 0) {
      o.err[r] = e;
      o.row_type[r] = uint8_t(p.type);
      static_cast<uint64_t *>(o.values)[r] = v;
      errs += e != 0;
    }
  }
  add_errors(s.tot, errs);
}

__global__ void __launch_bounds__(ptr::kCtaWarps * 32) col_size_cta_kernel(Cols c, int kind, Out o, Scratch s) {
  __shared__ ptr::CtaSmem<ptr::kCtaWarps> sm;
  ptr::CtaGroup<ptr::kCtaWarps> g{threadIdx.x, &sm};
  const uint32_t count = *s.list_count;
  for (uint32_t j = blockIdx.x; j < count; j += gridDim.x) {
    SizeAt at = s.handed[j];
    const uint32_t r = s.list_rows[j];
    count_children<ptr::CtaGroup<ptr::kCtaWarps>, ptr::kCtaItems>(g, c.type, c.n, kind == kObjectSize, &at, ~0ull);
    if (threadIdx.x == 0) {
      o.err[r] = 0;
      o.row_type[r] = uint8_t(kind == kObjectSize ? '{' : '[');
      static_cast<uint64_t *>(o.values)[r] = at.count < kCountSat ? at.count : kCountSat;
    }
  }
}

// ---- STRING
__device__ __forceinline__ unsigned long long block_sum(unsigned long long v, unsigned long long *sh) {
  for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, d);
  __syncthreads();
  if ((threadIdx.x & 31u) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long t = 0;
  for (int w = 0; w < kTile / 32; w++) t += sh[w];
  return t;
}

// the row checks; the length of row r goes to offsets[r + 1] until col_string_copy_kernel puts the offset there
__global__ void __launch_bounds__(kTile) col_string_len_kernel(Cols c, Out o, Scratch s) {
  __shared__ unsigned long long sh[kTile / 32];
  const uint32_t r = blockIdx.x * uint32_t(kTile) + threadIdx.x;
  uint64_t len = 0;
  uint32_t bad = 0;
  if (r < c.nrows) {
    const Pick p = pick_row(c, r);
    int32_t e = p.err;
    uint32_t t = p.type;
    if (e == 0) {
      uint64_t off;
      uint32_t l;
      if (t != '"') {
        e = kIncorrectType;
      } else if (!string_record(c, p.k, &off, &l)) {
        e = kUnexpectedError;
        t = 0;
      } else {
        len = l;
      }
    }
    o.err[r] = e;
    o.row_type[r] = uint8_t(t);
    o.offsets[uint64_t(r) + 1] = int64_t(len);
    bad = e != 0;
  }
  const unsigned long long tb = block_sum(len, sh);
  const unsigned long long te = block_sum(bad, sh);
  if (threadIdx.x == 0) {
    s.tile_sums[blockIdx.x] = tb;
    s.tile_errs[blockIdx.x] = uint32_t(te);
  }
}

// the offsets, then (when the column fits bytes_capacity) the copy.  A tile whose bytes fit kOutBytes composes them in
// shared memory at the destination's phase and writes them as aligned vectors; otherwise a lane copies a string of up to
// kLaneBytes, the warp one of up to kWarpBytes (group_copy), and longer ones are listed for col_string_long_kernel,
// one entry per kChunk bytes, written by the warp after one atomicAdd per string.
__global__ void __launch_bounds__(kTile) col_string_copy_kernel(Cols c, Out o, Scratch s, uint32_t ntiles) {
  __shared__ __align__(16) uint8_t outb[kOutBytes + 16];
  __shared__ unsigned long long sh[kTile / 32];
  const uint32_t r = blockIdx.x * uint32_t(kTile) + threadIdx.x;
  const unsigned lane = threadIdx.x & 31u;
  const uint64_t len = r < c.nrows ? uint64_t(o.offsets[uint64_t(r) + 1]) : 0;
  unsigned long long x = len;
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
    if (int(lane) >= d) x += y;
  }
  if (lane == 31) sh[threadIdx.x >> 5] = x;
  __syncthreads();
  unsigned long long rel = x - len;  // bytes of this tile's rows before mine
  for (uint32_t w = 0; w < (threadIdx.x >> 5); w++) rel += sh[w];
  const unsigned long long t_off = s.tile_sums[blockIdx.x];
  const unsigned long long total = s.tot->string_bytes;
  if (r < c.nrows) o.offsets[uint64_t(r) + 1] = int64_t(t_off + rel + len);
  if (r == 0) o.offsets[0] = 0;
  if (total > o.capacity) return;  // CAPACITY: offsets only
  const unsigned long long t_bytes = (blockIdx.x + 1 < ntiles ? s.tile_sums[blockIdx.x + 1] : total) - t_off;
  if (t_bytes == 0) return;  // (uniform)
  const uint8_t *src = len ? c.strbuf + c.payload[c.rows[r].index] + 4 : nullptr;
  uint8_t *dst_tile = o.bytes + t_off;
  const uint32_t phase = uint32_t(reinterpret_cast<uintptr_t>(dst_tile) & 15u);
  const bool staged = t_bytes <= kOutBytes;
  uint8_t *dst = staged ? outb + phase + rel : dst_tile + rel;
  if (len && len <= kLaneBytes)
    for (uint32_t i = 0; i < uint32_t(len); i++) dst[i] = src[i];
  const bool by_warp = len > kLaneBytes && (staged || len <= kWarpBytes);  // (a staged tile holds no string over kOutBytes)
  uint32_t listed = __ballot_sync(0xFFFFFFFFu, !staged && len > kWarpBytes);
  while (listed) {
    const int l = __ffs(int(listed)) - 1;
    listed &= listed - 1;
    const unsigned long long row = __shfl_sync(0xFFFFFFFFu, (unsigned long long)r, l);
    const uint32_t chunks = uint32_t((__shfl_sync(0xFFFFFFFFu, len, l) + kChunk - 1) / kChunk);
    uint32_t base = lane == 0 ? atomicAdd(s.list_count, chunks) : 0u;
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    for (uint32_t k = lane; k < chunks; k += 32) s.chunks[base + k] = (row << 32) | k;
  }
  uint32_t pending = __ballot_sync(0xFFFFFFFFu, by_warp);
  while (pending) {
    const int l = __ffs(int(pending)) - 1;
    pending &= pending - 1;
    uint8_t *d = reinterpret_cast<uint8_t *>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(dst), l));
    const uint8_t *sp = reinterpret_cast<const uint8_t *>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(src), l));
    const unsigned long long n = __shfl_sync(0xFFFFFFFFu, len, l);
    group_copy(lane, 32, d, sp, n);
  }
  if (!staged) return;
  __syncthreads();
  const uint32_t nb = uint32_t(t_bytes);
  const uint32_t head = (nb < ((16u - phase) & 15u)) ? nb : ((16u - phase) & 15u);
  const uint32_t nvec = (nb - head) >> 4;
  const uint32_t tail = nb - head - (nvec << 4);
  if (threadIdx.x < head) dst_tile[threadIdx.x] = outb[phase + threadIdx.x];
  const uint4 *sv = reinterpret_cast<const uint4 *>(outb + phase + head);  // (phase + head) % 16 == 0
  uint4 *gv = reinterpret_cast<uint4 *>(dst_tile + head);
  for (uint32_t v = threadIdx.x; v < nvec; v += kTile) gv[v] = sv[v];
  if (threadIdx.x < tail) dst_tile[head + (nvec << 4) + threadIdx.x] = outb[phase + head + (nvec << 4) + threadIdx.x];
}

// the strings over kWarpBytes: one CTA per listed chunk (grid-stride), so a long string is copied by many CTAs at once and
// a CTA reads only the entries it copies
__global__ void __launch_bounds__(kTile) col_string_long_kernel(Cols c, Out o, Scratch s) {
  const uint32_t count = *s.list_count;
  for (uint32_t j = blockIdx.x; j < count; j += gridDim.x) {
    const unsigned long long w = s.chunks[j];
    const uint32_t r = uint32_t(w >> 32);
    const uint64_t b = uint64_t(uint32_t(w)) * kChunk;
    const uint64_t at = uint64_t(o.offsets[r]), len = uint64_t(o.offsets[uint64_t(r) + 1]) - at;
    const uint8_t *src = c.strbuf + c.payload[c.rows[r].index] + 4;
    group_copy(threadIdx.x, kTile, o.bytes + at + b, src + b, len - b < kChunk ? len - b : kChunk);
  }
}

unsigned grid_of(uint64_t blocks, int sm_count, int per_sm) { return unsigned(blocks < uint64_t(sm_count) * per_sm ? (blocks ? blocks : 1) : uint64_t(sm_count) * per_sm); }

size_t align8(size_t b) { return (b + 7) & ~size_t(7); }

}  // namespace

size_t column_scratch_bytes(uint32_t nrows, uint64_t bytes_capacity) {
  const size_t tiles = (size_t(nrows) + kTile - 1) / kTile;
  return align8(sizeof(TokenTotals)) + 8 + align8(tiles * 8) + align8(tiles * 4) + align8(size_t(nrows) * sizeof(SizeAt)) + align8(size_t(nrows) * 4) +
         8 * long_chunk_capacity(bytes_capacity);
}

cudaError_t launch_column(const ColLaunch &a, void *scratch, TokenTotals **tot_out, int sm_count, cudaStream_t st, int *launches) {
  const uint32_t nrows = a.c.nrows;
  const uint32_t tiles = uint32_t((size_t(nrows) + kTile - 1) / kTile);
  uint8_t *p = static_cast<uint8_t *>(scratch);
  Scratch s;
  s.tot = reinterpret_cast<TokenTotals *>(p);
  p += align8(sizeof(TokenTotals));
  s.list_count = reinterpret_cast<uint32_t *>(p);
  p += 8;
  s.tile_sums = reinterpret_cast<unsigned long long *>(p);
  p += align8(size_t(tiles) * 8);
  s.tile_errs = reinterpret_cast<uint32_t *>(p);
  p += align8(size_t(tiles) * 4);
  s.handed = reinterpret_cast<SizeAt *>(p);
  p += align8(size_t(nrows) * sizeof(SizeAt));
  s.list_rows = reinterpret_cast<uint32_t *>(p);
  p += align8(size_t(nrows) * 4);
  s.chunks = reinterpret_cast<unsigned long long *>(p);
  *tot_out = s.tot;
  Out o{a.err, a.row_type, a.values, a.offsets, a.bytes, a.bytes_capacity};
  *launches = 0;
  cudaError_t e = cudaMemsetAsync(scratch, 0, align8(sizeof(TokenTotals)) + 8, st);
  if (e != cudaSuccess) return e;
  if (nrows == 0) {
    if (a.kind == kString) e = cudaMemsetAsync(a.offsets, 0, sizeof(int64_t), st);
    return e;
  }
  if (a.kind == kString) {
    col_string_len_kernel<<<tiles, kTile, 0, st>>>(a.c, o, s);
    e = launch_tile_scan(s.tile_sums, s.tile_errs, tiles, s.tot, st);
    if (e != cudaSuccess) return e;
    col_string_copy_kernel<<<tiles, kTile, 0, st>>>(a.c, o, s, tiles);
    col_string_long_kernel<<<unsigned(sm_count) * 4, kTile, 0, st>>>(a.c, o, s);
    *launches = 4;
  } else if (a.kind == kArraySize || a.kind == kObjectSize) {
    col_size_warp_kernel<<<grid_of((uint64_t(nrows) + 7) / 8, sm_count, 16), 256, 0, st>>>(a.c, a.kind, o, s);
    col_size_cta_kernel<<<unsigned(sm_count) * 2, ptr::kCtaWarps * 32, 0, st>>>(a.c, a.kind, o, s);
    *launches = 2;
  } else {
    col_scalar_kernel<<<grid_of((uint64_t(nrows) + 255) / 256, sm_count, 8), 256, 0, st>>>(a.c, a.kind, o, s);
    *launches = 1;
  }
  return cudaGetLastError();
}

}  // namespace col
}  // namespace sjb200
