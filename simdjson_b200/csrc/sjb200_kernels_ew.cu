// sjb200_kernels_ew.cu -- the emit-warp build of the stage-1 kernel (same source: sjb200_scan4.cuh), an option for large launches.
//
// Default build (sjb200_kernels.cu): a scan warp emits the block it scanned two iterations earlier (masks wait in shared
// memory).  This build: the 16 scan warps only scan, 7 more warps per CTA take resolved blocks from a CTA-wide queue
// and emit them; the masks wait in an L2-resident ring 8 elements deep, so a scan warp never waits for the chain.
// It pays off only for large launches (below, the ring fills before the first element is resolved, and at the end of a
// short launch only the emit is left to do): the host code picks this kernel for launches of at least `ew_min_bytes`
// (option; 0 = never, the default: on H100 this build was slower than the default one at every launch size from
// 256 MiB to 1 GiB, 13-16 % on NDJSON).
#ifdef SJB200_SCAN4_EMITW
#undef SJB200_SCAN4_EMITW
#endif
#ifdef SJB200_SCAN4_GPARK
#undef SJB200_SCAN4_GPARK
#endif
#define SJB200_SCAN4_EMITW 7
#define SJB200_SCAN4_GPARK 8
#include "sjb200_kernels.cuh"

#include "sjb200_bits.cuh"
#include "sjb200_scan4.cuh"

namespace sjb200 {

__global__ void __launch_bounds__(scan4::kThreads4, 1) scan4_ew_kernel(const __grid_constant__ CUtensorMap tmap, const ScanParams p) {
  extern __shared__ uint8_t smem_raw4e[];
  scan4::scan4_body<0>(&tmap, p, smem_raw4e, sj_smem_u32(smem_raw4e));
}

cudaError_t launch_scan4_ew(const CUtensorMap *tmap, const ScanParams &p, int grid, cudaStream_t stream) {
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(scan4_ew_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, scan4::kSmemBytes4);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  scan4_ew_kernel<<<grid, scan4::kThreads4, scan4::kSmemBytes4, stream>>>(*tmap, p);
  return cudaGetLastError();
}

size_t scan4_ew_park_words(int grid) { return size_t(grid) * scan4::kParkRing * scan4::kParkSlotWords + 8; }

}  // namespace sjb200
