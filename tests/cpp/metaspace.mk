# Host build of the SentencePiece-style BPE stages (smg_b200/csrc/metaspace.cuh, bpe.cuh) for tests/test_metaspace_host.py; needs no CUDA.
# Built by __graft_entry__.build():  make -C tests/cpp -f metaspace.mk
CXX ?= g++
CSRC := $(abspath ../..)/smg_b200/csrc
CXXFLAGS ?= -std=c++17 -O2 -Wall -Wextra -Wno-unused-parameter -Wno-unknown-pragmas

test_metaspace_host: test_metaspace_host.cpp $(CSRC)/metaspace.cuh $(CSRC)/bpe.cuh $(CSRC)/xxh3.cuh
	$(CXX) $(CXXFLAGS) -I$(CSRC) -o $@ $<
