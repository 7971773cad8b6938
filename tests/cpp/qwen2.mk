# Host build of the Qwen2 pre-tokenizer and the NFC normalizer (smg_b200/csrc/bpe.cuh, nfc.cuh) for tests/test_qwen2_host.py; needs no
# CUDA.  Built by __graft_entry__.build():  make -C tests/cpp -f qwen2.mk
CXX ?= g++
CSRC := $(abspath ../..)/smg_b200/csrc
CXXFLAGS ?= -std=c++17 -O2 -Wall -Wextra -Wno-unused-parameter -Wno-unknown-pragmas

test_qwen2_host: test_qwen2_host.cpp $(CSRC)/bpe.cuh $(CSRC)/nfc.cuh $(CSRC)/nfc_tables.h $(CSRC)/xxh3.cuh $(CSRC)/unicode_tables.h
	$(CXX) $(CXXFLAGS) -I$(CSRC) -o $@ $<
