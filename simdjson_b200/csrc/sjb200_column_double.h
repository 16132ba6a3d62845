// sjb200_column_double.h -- launcher of sjb200_column_double.cu (element::get_double of JSON Pointer results,
// sjb200_column_double_dev)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "sjb200_double.cuh"

namespace sjb200 {
namespace dbl {

struct DoubleLaunch {
  col::Cols c;          // the tokens and the rows (no string buffer)
  const uint8_t *buf;   // the input and its structurals (stage 1)
  uint64_t len;
  const uint32_t *idx;
  int32_t *err;
  uint8_t *row_type;
  uint64_t *values;     // the doubles' bits
};

// device scratch of a call over nrows rows, 8-byte aligned
size_t column_double_scratch_bytes(uint32_t nrows);
// The kernels on st, no synchronisation.  *rows_in_error: in the scratch, after the launches the rows in error.
cudaError_t launch_column_double(const DoubleLaunch &a, void *scratch, uint32_t **rows_in_error, int sm_count, cudaStream_t st, int *launches);

}  // namespace dbl
}  // namespace sjb200
