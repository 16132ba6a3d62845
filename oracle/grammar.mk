# oracle/grammar.mk -- builds the stage-2 grammar checkers.  TEST INFRASTRUCTURE ONLY.
#
#   libsj_grammar_oracle.so   : our C restatement of json_iterator::walk_document (sj_grammar_oracle.c); always buildable.
#   _ref/libsj_ref_grammar.so : the UNMODIFIED reference, compiled from the sources where they lie under $(REF) (no reference
#                               source enters this repo), plus ref_grammar_driver.cpp.  Only built when $(REF) is readable;
#                               the tests that use it are skipped without it.
REF ?= /root/reference
CC ?= gcc
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all: $(HERE)libsj_grammar_oracle.so ref

$(HERE)libsj_grammar_oracle.so: $(HERE)sj_grammar_oracle.c $(HERE)sj_grammar_oracle.h
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -Wextra -o $@ $(HERE)sj_grammar_oracle.c

ifneq ($(wildcard $(REF)/singleheader/simdjson.cpp),)
ref: $(HERE)_ref/libsj_ref_grammar.so
$(HERE)_ref/libsj_ref_grammar.so: $(HERE)ref_grammar_driver.cpp $(REF)/singleheader/simdjson.cpp $(REF)/singleheader/simdjson.h
	mkdir -p $(HERE)_ref
	$(CXX) -O2 -std=c++17 -fPIC -shared -fvisibility=hidden -Wl,-Bsymbolic \
	    -I$(REF)/singleheader -o $@ $(HERE)ref_grammar_driver.cpp $(REF)/singleheader/simdjson.cpp
else
ref:
	@echo "oracle: $(REF) not present; using prebuilt oracle/_ref if any"
endif

.PHONY: all ref
