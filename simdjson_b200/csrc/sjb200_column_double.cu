// sjb200_column_double.cu -- element::get_double of JSON Pointer results on the device (sjb200_column_double_dev): the
// routines of sjb200_double.cuh as sm_90a kernels.
//
//   dbl_row_kernel    one grid-stride pass, one thread per row: the row checks (col::pick_row), 'l' / 'u' rows, and 'd'
//                     rows of at most kLaneBytes bytes, summarized and converted by their lane.  A longer number is listed
//                     for dbl_long_kernel, an inconclusive one for dbl_exact_kernel (one atomicAdd each).
//   dbl_long_kernel   one CTA per listed long number (grid-stride): the CTA summarizes it; its first thread converts it,
//                     with the exact comparison when it is inconclusive.
//   dbl_exact_kernel  one thread per listed inconclusive row, the exact comparison on big integers in shared memory.
#include "sjb200_column_double.h"

#include "sjb200_pointer.h"

namespace sjb200 {
namespace dbl {
namespace {

constexpr uint32_t kLaneBytes = 64;  // a lane converts a number of at most this many bytes itself
constexpr int kExactThreads = 32;    // threads of a dbl_exact_kernel CTA (2 kLimbs words of shared memory each)

struct Scratch {  // column_double_scratch_bytes(nrows) bytes
  uint32_t *counts;     // [0] rows in error, [1] long numbers listed, [2] inconclusive rows listed
  uint32_t *long_rows;  // [nrows]
  uint32_t *slow_rows;  // [nrows]
};

struct Span {
  bool ok;  // inside [0, len) and not empty
  SpanSrc at;
};
__device__ __forceinline__ Span span_of(const DoubleLaunch &a, uint32_t k) {
  const uint64_t b0 = a.idx[k], b1 = a.c.payload[k];
  if (!(b0 < b1 && b1 <= a.len)) return Span{false, SpanSrc{nullptr, 0}};
  return Span{true, SpanSrc{a.buf + b0, uint32_t(b1 - b0)}};
}

__device__ __forceinline__ void put(const DoubleLaunch &a, uint32_t r, int32_t e, uint32_t t, uint64_t bits) {
  a.err[r] = e;
  a.row_type[r] = uint8_t(t);
  a.values[r] = e ? 0u : bits;
}

__global__ void __launch_bounds__(256) dbl_row_kernel(DoubleLaunch a, Scratch s) {
  uint32_t errs = 0;
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t r = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; r < a.c.nrows; r += stride) {
    const col::Pick p = col::pick_row(a.c, uint32_t(r));
    int32_t e = p.err;
    uint32_t t = p.type;
    uint64_t bits = 0;
    if (e == 0) {
      if (t == 'l' || t == 'u') {
        bits = integer_bits(t, a.c.payload[p.k]);
      } else if (t != 'd') {
        e = ptr::kIncorrectType;
      } else {
        const Span sp = span_of(a, p.k);
        if (!sp.ok) {
          e = ptr::kUnexpectedError;
          t = 0;
        } else if (sp.at.len > kLaneBytes) {
          s.long_rows[atomicAdd(&s.counts[1], 1u)] = uint32_t(r);
          continue;  // written by dbl_long_kernel
        } else {
          SerialGroup g;
          const Num m = summarize(g, sp.at, sp.at.len);
          uint64_t fb;
          if (!m.valid) {
            e = ptr::kUnexpectedError;
            t = 0;
          } else if ((e = convert(m, sp.at, &bits, &fb)) == kSlow) {
            s.slow_rows[atomicAdd(&s.counts[2], 1u)] = uint32_t(r);
            continue;  // written by dbl_exact_kernel
          }
        }
      }
    }
    put(a, uint32_t(r), e, t, bits);
    errs += e != 0;
  }
  const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, errs);
  if ((threadIdx.x & 31u) == 0 && w) atomicAdd(&s.counts[0], w);
}

__global__ void __launch_bounds__(ptr::kCtaWarps * 32) dbl_long_kernel(DoubleLaunch a, Scratch s) {
  __shared__ ptr::CtaSmem<ptr::kCtaWarps> sm;
  __shared__ uint32_t big[2 * kLimbs];
  ptr::CtaGroup<ptr::kCtaWarps> g{threadIdx.x, &sm};
  const uint32_t count = s.counts[1];
  for (uint32_t j = blockIdx.x; j < count; j += gridDim.x) {
    const uint32_t r = s.long_rows[j];
    const Span sp = span_of(a, a.c.rows[r].index);  // (checked by dbl_row_kernel)
    const Num m = summarize(g, sp.at, sp.at.len);
    if (threadIdx.x != 0) continue;
    int32_t e = ptr::kUnexpectedError;
    uint32_t t = 0;
    uint64_t bits = 0, fb = 0;
    if (m.valid) {
      t = 'd';
      e = convert(m, sp.at, &bits, &fb);
      if (e == kSlow) e = finish_exact(m, exact(m, sp.at, fb, Big{big, 1, 0}, Big{big + kLimbs, 1, 0}), &bits);
    }
    put(a, r, e, t, bits);
    if (e) atomicAdd(&s.counts[0], 1u);
  }
}

__global__ void __launch_bounds__(kExactThreads) dbl_exact_kernel(DoubleLaunch a, Scratch s) {
  __shared__ uint32_t big[2 * kLimbs * kExactThreads];  // limb i of thread t's numbers at [i * kExactThreads + t]
  const uint32_t count = s.counts[2];
  uint32_t errs = 0;
  for (uint32_t j = blockIdx.x * kExactThreads + threadIdx.x; j < count; j += gridDim.x * kExactThreads) {
    const uint32_t r = s.slow_rows[j];
    const Span sp = span_of(a, a.c.rows[r].index);  // (checked by dbl_row_kernel)
    SerialGroup g;
    const Num m = summarize(g, sp.at, sp.at.len);
    uint64_t bits = 0, fb = 0;
    int32_t e = convert(m, sp.at, &bits, &fb);
    if (e == kSlow)
      e = finish_exact(m, exact(m, sp.at, fb, Big{big + threadIdx.x, kExactThreads, 0}, Big{big + kLimbs * kExactThreads + threadIdx.x, kExactThreads, 0}),
                       &bits);
    put(a, r, e, 'd', bits);
    errs += e != 0;
  }
  if (errs) atomicAdd(&s.counts[0], errs);
}

unsigned grid_of(uint64_t blocks, int sm_count, int per_sm) { return unsigned(blocks < uint64_t(sm_count) * per_sm ? (blocks ? blocks : 1) : uint64_t(sm_count) * per_sm); }

}  // namespace

size_t column_double_scratch_bytes(uint32_t nrows) { return 16 + 8 * size_t(nrows); }

cudaError_t launch_column_double(const DoubleLaunch &a, void *scratch, uint32_t **rows_in_error, int sm_count, cudaStream_t st, int *launches) {
  const uint32_t nrows = a.c.nrows;
  uint8_t *p = static_cast<uint8_t *>(scratch);
  Scratch s;
  s.counts = reinterpret_cast<uint32_t *>(p);
  s.long_rows = reinterpret_cast<uint32_t *>(p + 16);
  s.slow_rows = s.long_rows + nrows;
  *rows_in_error = s.counts;
  *launches = 0;
  cudaError_t e = cudaMemsetAsync(scratch, 0, 16, st);
  if (e != cudaSuccess || nrows == 0) return e;
  dbl_row_kernel<<<grid_of((uint64_t(nrows) + 255) / 256, sm_count, 8), 256, 0, st>>>(a, s);
  dbl_long_kernel<<<unsigned(sm_count) * 2, ptr::kCtaWarps * 32, 0, st>>>(a, s);
  dbl_exact_kernel<<<unsigned(sm_count) * 4, kExactThreads, 0, st>>>(a, s);
  *launches = 3;
  return cudaGetLastError();
}

}  // namespace dbl
}  // namespace sjb200
