// sjb200_kernels.cuh -- shared declarations between the kernels and the C-ABI host code.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "sjb200_common.h"
#include "sjb200_params.h"

namespace sjb200 {

// launchers (defined in sjb200_kernels.cu)
// scan4: the stage-1 indexer of sjb200_scan4.cuh (4 KiB blocks; its tensor map has a 32-row box).  pdl (stage 1 only):
// programmatic dependent launch -- the kernel may start while the previous operation on the stream, a scan4 stage-1
// launch, is still running (ScanParams::early_input)
cudaError_t launch_scan4(const CUtensorMap *tmap, const ScanParams &p, int grid, int mode /*0 stage 1, 2 minify*/,
                         cudaStream_t stream, bool pdl = false);
int scan4_tiles_per_element();      // 32 KiB tiles of the launch parameter block per scan4 element
int scan4_max_ctas_per_sm();
constexpr int kScan4BoxRows = 32;
// utf8v2: validate_utf8 with independent warps (sjb200_utf8.cuh); same 32-row boxes
cudaError_t launch_utf8v2(const CUtensorMap *tmap, const ScanParams &p, int grid, cudaStream_t stream);
int utf8v2_max_ctas_per_sm();
int utf8v2_warps_per_cta();
cudaError_t launch_gather_tails(const uint8_t *const *bufs, const uint64_t *lens, uint32_t ndocs, uint8_t *out, cudaStream_t stream);
// republish a shard record {w0, w1} in every rank's exchange window (x)
cudaError_t launch_xchg_post(const Xchg &x, unsigned long long w0, unsigned long long w1, cudaStream_t stream);
cudaError_t launch_write_sentinels(uint32_t *idx, uint32_t n, uint32_t a, uint32_t b, uint32_t c, cudaStream_t stream);

}  // namespace sjb200
