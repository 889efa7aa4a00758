# Build recipe for the perplexity oracle (TEST INFRASTRUCTURE, not product code).
#
#   make -C oracle -f perplexity.mk   -> oracle/_ref/libfalcon_ppl.so
#
# Compiles the reference's examples/falcon_perplexity/falcon_perplexity.cpp (its `main` renamed, so the program's own softmax and
# perplexity loop come along unchanged) and examples/falcon_common.cpp where they lie under $(REF), and links them with the reference
# objects of `make -C oracle ref` and ref_perplexity.cpp, which exports the reference's softmax to ctypes.  The program includes a
# build-info.h that the reference's own Makefile generates; a stand-in is written under _ref/.  Same flags as the `ref` target.
REF      ?= /root/reference
CXX      ?= g++
ARCH     ?= -march=x86-64-v3
REFDEFS   = -DGGML_USE_K_QUANTS -D_GNU_SOURCE -D_XOPEN_SOURCE=600 -DNDEBUG -DGGML_PERF=1
CXXFLAGS_R= -O3 -std=c++11 -fPIC $(ARCH) -pthread $(REFDEFS) -I$(REF) -I$(REF)/examples -w

all: _ref/libfalcon_ppl.so

_ref/build-info.h:
	printf '#define BUILD_NUMBER 0\n#define BUILD_COMMIT "oracle"\n' > $@
_ref/falcon_perplexity.o: $(REF)/examples/falcon_perplexity/falcon_perplexity.cpp _ref/build-info.h
	$(CXX) $(CXXFLAGS_R) -I_ref -Dmain=falcon_perplexity_main -c $< -o $@
_ref/falcon_common.o: $(REF)/examples/falcon_common.cpp
	$(CXX) $(CXXFLAGS_R) -c $< -o $@
# remade on every build, like sample_chain.mk's harness: a prebuilt _ref copied into a checkout is newer than its sources
_ref/ref_perplexity.o: ref_perplexity.cpp FORCE
	$(CXX) $(CXXFLAGS_R) -c $< -o $@
_ref/libfalcon_ppl.so: _ref/ggml.o _ref/k_quants.o _ref/libfalcon.o _ref/cmpnct_unicode.o _ref/falcon_common.o _ref/falcon_perplexity.o _ref/ref_perplexity.o FORCE
	$(CXX) -shared -o $@ $(filter %.o,$^) -lm -pthread

FORCE:
.PHONY: all FORCE
