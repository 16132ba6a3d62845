# oracle/double.mk -- builds the get_double checkers.  TEST INFRASTRUCTURE ONLY.
#
#   libsj_double_oracle.so   : our C restatement of element::get_double on a JSON Pointer result (sj_double_oracle.c);
#                              always buildable.
#   _ref/libsj_ref_double.so : the UNMODIFIED reference, compiled from the sources where they lie under $(REF) (no
#                              reference source enters this repo), plus ref_double_driver.cpp.  Only built when $(REF) is
#                              readable; the tests that use it are skipped without it.
REF ?= /root/reference
CC ?= gcc
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all: $(HERE)libsj_double_oracle.so ref

$(HERE)libsj_double_oracle.so: $(HERE)sj_double_oracle.c
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -Wextra -o $@ $(HERE)sj_double_oracle.c

ifneq ($(wildcard $(REF)/singleheader/simdjson.cpp),)
ref: $(HERE)_ref/libsj_ref_double.so
$(HERE)_ref/libsj_ref_double.so: $(HERE)ref_double_driver.cpp $(REF)/singleheader/simdjson.cpp $(REF)/singleheader/simdjson.h
	mkdir -p $(HERE)_ref
	$(CXX) -O2 -std=c++17 -fPIC -shared -fvisibility=hidden -Wl,-Bsymbolic \
	    -I$(REF)/singleheader -o $@ $(HERE)ref_double_driver.cpp $(REF)/singleheader/simdjson.cpp
else
ref:
	@echo "oracle: $(REF) not present; using prebuilt oracle/_ref if any"
endif

.PHONY: all ref
