// sjb200_pointer.h -- launcher of sjb200_pointer.cu (JSON Pointer lookup, sjb200_at_pointer_dev)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_docs.h"
#include "sjb200_pointer.cuh"

namespace sjb200 {
namespace ptr {

// A document of more structurals than this is walked by a CTA of kCtaWarps warps, kCtaItems structurals per thread per
// step; one of at most this many by a warp, one structural per lane per step (DESIGN.md section 4.6).
#ifndef SJB200_POINTER_CTA_MIN
#define SJB200_POINTER_CTA_MIN 4096
#endif
constexpr uint32_t kCtaMinStructurals = SJB200_POINTER_CTA_MIN;
constexpr unsigned kCtaWarps = 8;
constexpr int kCtaItems = 8;

struct PtrResult {  // sjb200_pointer_result
  int32_t error;
  uint32_t index;
};

struct PtrLaunch {
  Walk w;
  uint32_t n;
  const sjb200_doc_boundary_t *docs;  // null: one document [0, n)
  uint32_t ndocs;
  const PtrHeader *headers;
  uint32_t npointers;
  PtrResult *out;  // [npointers][docs ? ndocs : 1]
  // scratch, set by launch_at_pointer
  uint32_t *long_count, *first_err, *long_docs;
};

size_t pointer_scratch_words(uint32_t ndocs);
// scratch: pointer_scratch_words(ndocs) words of device memory.  Three launches on s, no synchronisation.
cudaError_t launch_at_pointer(const PtrLaunch &a, uint32_t *scratch, int sm_count, cudaStream_t s);

}  // namespace ptr
}  // namespace sjb200
