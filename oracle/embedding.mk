# Build recipe for the embedding oracle (TEST INFRASTRUCTURE, not product code).
#
#   make -C oracle -f embedding.mk   -> oracle/_ref/libfalcon_emb.so, oracle/_ref/libfalcon_hook_emb.so
#
# Needs the reference objects of `make -C oracle ref` (the reference sources read in place under $(REF)); links them with
# ref_harness.cpp (eval, free) and ref_embedding.cpp (a context loaded with embedding = true), once for the CPU build and once for
# the -DGGML_USE_CUBLAS build whose ggml_cuda_* symbols libggml_b200.so provides.  Same flags as the `ref` target.
REF      ?= /root/reference
CXX      ?= g++
ARCH     ?= -march=x86-64-v3
REFDEFS   = -DGGML_USE_K_QUANTS -D_GNU_SOURCE -D_XOPEN_SOURCE=600 -DNDEBUG -DGGML_PERF=1
CXXFLAGS_R= -O3 -std=c++11 -fPIC $(ARCH) -pthread $(REFDEFS) -I$(REF) -I$(REF)/examples -w
CUDA_INC ?= /usr/local/cuda/include

all: _ref/libfalcon_emb.so _ref/libfalcon_hook_emb.so

# remade on every build, like sample_chain.mk's harness: a prebuilt _ref copied into a checkout is newer than its sources
_ref/ref_embedding.o: ref_embedding.cpp FORCE
	$(CXX) $(CXXFLAGS_R) -c $< -o $@
_ref/ref_embedding_hook.o: ref_embedding.cpp FORCE
	$(CXX) $(CXXFLAGS_R) -DGGML_USE_CUBLAS -I$(CUDA_INC) -c $< -o $@
_ref/libfalcon_emb.so: _ref/ggml.o _ref/k_quants.o _ref/libfalcon.o _ref/cmpnct_unicode.o _ref/ref_harness.o _ref/ref_embedding.o FORCE
	$(CXX) -shared -o $@ $(filter %.o,$^) -lm -pthread
_ref/libfalcon_hook_emb.so: _ref/ggml_hook.o _ref/k_quants.o _ref/libfalcon_hook.o _ref/cmpnct_unicode.o _ref/ref_harness_hook.o _ref/ref_embedding_hook.o FORCE
	$(CXX) -shared -o $@ $(filter %.o,$^) -lm -pthread

FORCE:
.PHONY: all FORCE
