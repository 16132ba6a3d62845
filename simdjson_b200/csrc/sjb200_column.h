// sjb200_column.h -- launcher of sjb200_column.cu (typed columns from JSON Pointer results, sjb200_column_dev)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_column.cuh"
#include "sjb200_tape.h"

namespace sjb200 {
namespace col {

struct ColLaunch {
  Cols c;
  int kind;
  int32_t *err;
  uint8_t *row_type;
  void *values;             // not STRING: uint64 (INT64 as its bits, UINT64, the sizes) or uint8 (BOOL) per row
  int64_t *offsets;         // STRING: nrows + 1
  uint8_t *bytes;           // STRING: bytes_capacity
  uint64_t bytes_capacity;
};

// device scratch of a call over nrows rows into a.bytes of bytes_capacity bytes (0 but for STRING), 8-byte aligned
size_t column_scratch_bytes(uint32_t nrows, uint64_t bytes_capacity);
// The kernels of a.kind on st, no synchronisation.  *tot: in the scratch, after the launches n_strings holds the rows in
// error and (STRING) string_bytes the column's bytes; nothing is written to a.bytes when they exceed a.bytes_capacity.
cudaError_t launch_column(const ColLaunch &a, void *scratch, TokenTotals **tot, int sm_count, cudaStream_t st, int *launches);

}  // namespace col
}  // namespace sjb200
