#!/bin/bash
# tuning aid: builds libsjb200 variants with different -D flags into tools/variants/ (select one with SJB200_LIB=...)
# usage: build_variants.sh name1 "flags1" name2 "flags2" ...   e.g. build_variants.sh park4 "-DSJB200_SCAN4_PARK=4"
set -e
cd "$(dirname "$0")/.."
if [ $# -lt 2 ]; then
  echo "usage: $0 name1 \"flags1\" [name2 \"flags2\" ...]" >&2
  exit 2
fi
# the library's sources, as the Makefile lists them
SRCS=$(make -s -C simdjson_b200/csrc --eval 'print-srcs: ; @echo $(SRCS)' print-srcs)
FLAGS="-O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fvisibility=hidden -shared"
mkdir -p tools/variants
rm -f tools/variants/*.so
build() { name=$1; shift; nvcc $FLAGS "$@" -o tools/variants/lib_$name.so $SRCS & }
while [ $# -gt 1 ]; do build "$1" $2; shift 2; done
wait
ls -la tools/variants
