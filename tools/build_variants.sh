#!/bin/bash
# tuning aid: builds libsjb200 variants with different -D flags into tools/variants/ (select one with SJB200_LIB=...)
set -e
cd "$(dirname "$0")/.."
SRCS="simdjson_b200/csrc/sjb200_kernels.cu simdjson_b200/csrc/sjb200_kernels_ew.cu simdjson_b200/csrc/sjb200_docs.cu simdjson_b200/csrc/sjb200_capi.cu simdjson_b200/csrc/sjb200_finish.cpp simdjson_b200/csrc/sjb200_hostcopy.cpp"
FLAGS="-O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fvisibility=hidden -shared"
mkdir -p tools/variants
rm -f tools/variants/*.so
build() { name=$1; shift; nvcc $FLAGS "$@" -o tools/variants/lib_$name.so $SRCS & }
if [ $# -gt 0 ]; then
  # usage: build_variants.sh name1 "flags1" name2 "flags2" ...
  while [ $# -gt 1 ]; do build "$1" $2; shift 2; done
else
  build emit0 -DSJB200_SCAN4_EMIT=0
  build emit1 -DSJB200_SCAN4_EMIT=1
  build emit2 -DSJB200_SCAN4_EMIT=2
  build emit1_park4 -DSJB200_SCAN4_EMIT=1 -DSJB200_SCAN4_PARK=4
  build emit1_stag -DSJB200_SCAN4_EMIT=1 -DSJB200_SCAN4_PARK=4 -DSJB200_SCAN4_STAGGER=1
  build emit0_stag -DSJB200_SCAN4_EMIT=0 -DSJB200_SCAN4_PARK=4 -DSJB200_SCAN4_STAGGER=1
  build emit1_counter -DSJB200_SCAN4_EMIT=1 -DSJB200_SCAN4_COUNTER=1
  build diag_noutf8 -DSJB200_SCAN4_EMIT=1 -DSJB200_DIAG_NO_UTF8
  build diag_noemit -DSJB200_SCAN4_EMIT=1 -DSJB200_DIAG_NO_EMIT
fi
wait
ls -la tools/variants
