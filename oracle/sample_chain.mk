# Build recipe for the whole-chain sampling oracle (TEST INFRASTRUCTURE, not product code).
#
#   make -C oracle -f sample_chain.mk   -> oracle/_ref/libfalcon_chain.so
#
# Needs the reference objects of `make -C oracle ref` (the reference sources read in place under $(REF)); links them with
# ref_harness.cpp (context handle, seeding) and ref_sample_chain.cpp (falcon_main's whole chain).  Same flags as the `ref` target.
REF      ?= /root/reference
CXX      ?= g++
ARCH     ?= -march=x86-64-v3
REFDEFS   = -DGGML_USE_K_QUANTS -D_GNU_SOURCE -D_XOPEN_SOURCE=600 -DNDEBUG -DGGML_PERF=1
CXXFLAGS_R= -O3 -std=c++11 -fPIC $(ARCH) -pthread $(REFDEFS) -I$(REF) -I$(REF)/examples -w

all: _ref/libfalcon_chain.so

_ref/ref_sample_chain.o: ref_sample_chain.cpp
	$(CXX) $(CXXFLAGS_R) -c $< -o $@
_ref/libfalcon_chain.so: _ref/ggml.o _ref/k_quants.o _ref/libfalcon.o _ref/cmpnct_unicode.o _ref/ref_harness.o _ref/ref_sample_chain.o
	$(CXX) -shared -o $@ $^ -lm -pthread

.PHONY: all
