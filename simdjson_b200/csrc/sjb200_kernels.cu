// sjb200_kernels.cu -- the sm_90a kernels' entry points and launchers.
//
// What the kernels replace in the reference (CPU, 64-byte SIMD blocks, strictly serial carries):
//   json_structural_indexer::index<128> / step / next   src/generic/stage1/json_structural_indexer.h L193-247
//   json_scanner::next, json_string_scanner::next, json_escape_scanner::next
//                                                        json_scanner.h L134-157, json_string_scanner.h L62-85,
//                                                        json_escape_scanner.h L50-71
//   bit_indexer::write                                   json_structural_indexer.h L93-122 (src/icelake.cpp L129-160)
//   utf8_checker                                         utf8_lookup4_algorithm.h L145-202
//   json_minifier::minify<128>                           json_minifier.h L68-97
//   generic_validate_utf8                                utf8_validator.h L18-34
//
// The kernel bodies live in headers written against the small primitive set of sjb200_simt.cuh (so that the same source
// runs under the host SIMT emulation, tests/simt_emul.cpp):
//   sjb200_scan4.cuh   stage 1 (structural indexing + UTF-8 validation) and minify: 4 KiB blocks by TMA, warp-independent
//                      both-polarity block scans, one decoupled look-back chain, per-lane bit-loop emit
//   sjb200_utf8.cuh    validate_utf8: independent warps, no chain
//   sjb200_bits.cuh    the bit-plane algebra both use
#include "sjb200_kernels.cuh"

#include "sjb200_bits.cuh"
#include "sjb200_scan4.cuh"
#include "sjb200_utf8.cuh"

namespace sjb200 {

// ------------------------------------------------------------------ scan4 (stage 1; see sjb200_scan4.cuh)
// two variants of one source: pipelined (masks wait in shared memory, an element is emitted two scans after it was scanned)
// and deferred (masks wait in an L2-resident scratch ring, everything is emitted after the CTA's last scan: launches
// small enough that every CTA holds all its elements at once never stall on the chain)
__global__ void __launch_bounds__(scan4::kThreads4, (SJB200_SCAN4_WARPS > 8) ? 1 : SJB200_SCAN4_MIN_CTAS)
    scan4_kernel(const __grid_constant__ CUtensorMap tmap, const ScanParams p) {
  extern __shared__ uint8_t smem_raw4[];
  scan4::scan4_body<0>(&tmap, p, smem_raw4, sj_smem_u32(smem_raw4));
}
__global__ void __launch_bounds__(scan4::kThreads4, (SJB200_SCAN4_WARPS > 8) ? 1 : SJB200_SCAN4_MIN_CTAS)
    scan4_minify_kernel(const __grid_constant__ CUtensorMap tmap, const ScanParams p) {
  extern __shared__ uint8_t smem_raw4[];
  scan4::scan4_body<2>(&tmap, p, smem_raw4, sj_smem_u32(smem_raw4));
}

// validate_utf8, every warp on its own (sjb200_utf8.cuh)
__global__ void __launch_bounds__(utf8v2::kThreadsU, utf8v2::kCtasPerSmU)
    utf8v2_kernel(const __grid_constant__ CUtensorMap tmap, const ScanParams p) {
  extern __shared__ uint8_t smem_raw_u[];
  utf8v2::utf8_body(&tmap, p, smem_raw_u, sj_smem_u32(smem_raw_u));
}

// ------------------------------------------------------------------ small helpers
// last min(3, len) bytes of many device-resident documents into one small array (streaming modes trim a partial UTF-8
// tail before the scan: json_structural_indexer.h L198-204) -- one launch + one copy for a whole batch
__global__ void gather_tails_kernel(const uint8_t *const *bufs, const uint64_t *lens, uint32_t ndocs, uint8_t *out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ndocs) return;
  const uint64_t len = lens[i];
  const uint32_t k = len < 3 ? uint32_t(len) : 3u;
  for (uint32_t b = 0; b < 4; b++) out[4 * i + b] = (b < k) ? bufs[i][len - k + b] : 0;
}
__global__ void write_sentinels_kernel(uint32_t *idx, uint32_t n, uint32_t a, uint32_t b, uint32_t c) {
  idx[n] = a;
  idx[n + 1] = b;
  idx[n + 2] = c;
}

// second round of a sharded pass (after re-scans): republish this rank's record in every rank's exchange window
__global__ void xchg_post_kernel(ScanParams p, unsigned long long w0, unsigned long long w1) {
  const uint32_t r = threadIdx.x;
  if (r < p.xchg_nranks) {
    unsigned long long *rec = p.xchg_peer[r] + (size_t(p.xchg_slot) * kMaxRanks + p.xchg_rank) * 2;
    sj_st_sys_u64(rec, w0);
    sj_st_sys_u64(rec + 1, w1);
  }
}

// ------------------------------------------------------------------ launchers
cudaError_t launch_scan4(const CUtensorMap *tmap, const ScanParams &p, int grid, int mode, cudaStream_t stream) {
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(scan4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, scan4::kSmemBytes4);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(scan4_minify_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, scan4::kSmemBytes4);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  if (mode == 2) scan4_minify_kernel<<<grid, scan4::kThreads4, scan4::kSmemBytes4, stream>>>(*tmap, p);
  else scan4_kernel<<<grid, scan4::kThreads4, scan4::kSmemBytes4, stream>>>(*tmap, p);
  return cudaGetLastError();
}

cudaError_t launch_utf8v2(const CUtensorMap *tmap, const ScanParams &p, int grid, cudaStream_t stream) {
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(utf8v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, utf8v2::kSmemBytesU);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  utf8v2_kernel<<<grid, utf8v2::kThreadsU, utf8v2::kSmemBytesU, stream>>>(*tmap, p);
  return cudaGetLastError();
}
int utf8v2_max_ctas_per_sm() {
  int n = 0;
  cudaFuncSetAttribute(utf8v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, utf8v2::kSmemBytesU);
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, utf8v2_kernel, utf8v2::kThreadsU, utf8v2::kSmemBytesU);
  return (e == cudaSuccess && n > 0) ? n : 1;
}
int utf8v2_warps_per_cta() { return utf8v2::kWarpsU; }

size_t scan4_park_words(int grid) { return size_t(grid) * scan4::kParkRing * scan4::kParkSlotWords + 8; }
int scan4_parks_in_global() { return scan4::kGPark > 0 ? 1 : 0; }
int scan4_tiles_per_element() { return scan4::kElemBytes / kTileBytes; }

int scan4_max_ctas_per_sm() {
  int n = 0;
  cudaFuncSetAttribute(scan4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, scan4::kSmemBytes4);
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, scan4_kernel, scan4::kThreads4, scan4::kSmemBytes4);
  return (e == cudaSuccess && n > 0) ? n : 1;
}

cudaError_t launch_gather_tails(const uint8_t *const *bufs, const uint64_t *lens, uint32_t ndocs, uint8_t *out, cudaStream_t stream) {
  if (ndocs == 0) return cudaSuccess;
  gather_tails_kernel<<<(ndocs + 127) / 128, 128, 0, stream>>>(bufs, lens, ndocs, out);
  return cudaGetLastError();
}

cudaError_t launch_xchg_post(const ScanParams &p, unsigned long long w0, unsigned long long w1, cudaStream_t stream) {
  xchg_post_kernel<<<1, 32, 0, stream>>>(p, w0, w1);
  return cudaGetLastError();
}

cudaError_t launch_write_sentinels(uint32_t *idx, uint32_t n, uint32_t a, uint32_t b, uint32_t c, cudaStream_t stream) {
  write_sentinels_kernel<<<1, 1, 0, stream>>>(idx, n, a, b, c);
  return cudaGetLastError();
}

}  // namespace sjb200
