# Host build of the DeepSeek pre-tokenizer (smg_b200/csrc/bpe.cuh on deepseek_tables.h) for tests/test_deepseek_host.py; needs no CUDA.
# Built by __graft_entry__.build():  make -C tests/cpp -f deepseek.mk
CXX ?= g++
CSRC := $(abspath ../..)/smg_b200/csrc
CXXFLAGS ?= -std=c++17 -O2 -Wall -Wextra -Wno-unused-parameter -Wno-unknown-pragmas

test_deepseek_host: test_deepseek_host.cpp $(CSRC)/bpe.cuh $(CSRC)/xxh3.cuh $(CSRC)/deepseek_tables.h
	$(CXX) $(CXXFLAGS) -I$(CSRC) -o $@ $<
