# consistent_hashing test programs, built by __graft_entry__.build():
#   make -C tests/cpp -f consistent_hashing.mk test_consistent_hashing libchash_oracle.so
# test_consistent_hashing: the C++ mirror smgx::ConsistentHashingPolicy (include/smgx.hpp over smg_b200/libsmgx.so); runs on the GPU.
CXX ?= g++
ROOT := $(abspath ../..)
CXXFLAGS ?= -std=c++17 -O2 -Wall -Wextra -Wno-unused-parameter

test_consistent_hashing: test_consistent_hashing.cpp $(ROOT)/include/smgx.hpp $(ROOT)/include/smgx.h $(ROOT)/smg_b200/libsmgx.so
	$(CXX) $(CXXFLAGS) -o $@ $< -L$(ROOT)/smg_b200 -lsmgx -Wl,-rpath,'$$ORIGIN/../../smg_b200'

# the CPU oracle (consistent_hashing_oracle.h) as a shared library for ctypes; needs no CUDA
ORACLE_FLAGS := -std=c++17 -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter -pthread
libchash_oracle.so: consistent_hashing_oracle.cc consistent_hashing_oracle.h $(ROOT)/oracle/prefix_hash.h $(ROOT)/oracle/power_of_two.h $(ROOT)/oracle/blake3_ref.h
	$(CXX) $(ORACLE_FLAGS) -shared -o $@ $<
