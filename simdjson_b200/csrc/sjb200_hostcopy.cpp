// sjb200_hostcopy.cpp -- the copy loop of the staging threads (sjb200_hostpipe.h): pageable source -> page-locked ring.
// Streaming (non-temporal) stores: the destination is about to be read by the copy engine, not by this core, and a
// plain memcpy of a sub-megabyte piece first READS every destination line (write-allocate), which halves what a thread
// moves.
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#if defined(__x86_64__)
#include <immintrin.h>

namespace {
__attribute__((target("avx2"))) void copy_avx2(uint8_t *dst, const uint8_t *src, size_t n) {
  size_t i = 0;
  for (; i + 128 <= n; i += 128) {
    const __m256i a = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i));
    const __m256i b = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i + 32));
    const __m256i c = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i + 64));
    const __m256i d = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i + 96));
    _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i), a);
    _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i + 32), b);
    _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i + 64), c);
    _mm256_stream_si256(reinterpret_cast<__m256i *>(dst + i + 96), d);
  }
  if (i < n) memcpy(dst + i, src + i, n - i);
  _mm_sfence();  // the streamed lines must be globally visible before the piece is reported done
}
}  // namespace
#endif

namespace sjb200 {

void copy_to_staging(void *dst, const void *src, size_t n) {
#if defined(__x86_64__)
  static const bool avx2 = __builtin_cpu_supports("avx2");
  if (avx2 && (reinterpret_cast<uintptr_t>(dst) & 31u) == 0 && n >= 4096) {
    copy_avx2(static_cast<uint8_t *>(dst), static_cast<const uint8_t *>(src), n);
    return;
  }
#endif
  memcpy(dst, src, n);
}

}  // namespace sjb200
