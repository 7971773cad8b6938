# Host build of the r50k pre-tokenizer (smg_b200/csrc/bpe.cuh) for tests/test_r50k_splitter.py; needs no CUDA.  Built by
# __graft_entry__.build():  make -C tests/cpp -f splitter.mk
CXX ?= g++
ROOT := $(abspath ../..)
CSRC := $(ROOT)/smg_b200/csrc
CXXFLAGS ?= -std=c++17 -O2 -Wall -Wextra -Wno-unused-parameter -Wno-unknown-pragmas

test_r50k_splitter: test_r50k_splitter.cpp $(CSRC)/bpe.cuh $(CSRC)/xxh3.cuh $(CSRC)/unicode_tables.h
	$(CXX) $(CXXFLAGS) -I$(CSRC) -o $@ $<
