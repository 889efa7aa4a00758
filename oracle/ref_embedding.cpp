// ref_embedding.cpp -- a context of the UNMODIFIED reference with falcon_context_params.embedding set (libfalcon.h:108), for ctypes.
//
// TEST INFRASTRUCTURE ONLY.  Built by oracle/embedding.mk into oracle/_ref/libfalcon_emb.so (CPU build) and
// oracle/_ref/libfalcon_hook_emb.so (-DGGML_USE_CUBLAS build, the operator hook) together with the reference objects and
// ref_harness.cpp, whose refh_eval / refh_free drive the context.  The row itself is read with the reference's own
// falcon_get_embeddings (libfalcon.h:267) through ctypes; no arithmetic here.
#include "libfalcon.h"

extern "C" {

// refh_load (ref_harness.cpp) plus `embedding`: every falcon_eval then also copies the last row of "result_norm" into the context
void * refh_load_ex(const char * path, int n_ctx, int n_batch, int n_gpu_layers, int logits_all, int embedding) {
    static bool backend_ready = false;
    if (!backend_ready) { falcon_init_backend(); backend_ready = true; }
    falcon_context_params p = falcon_context_default_params();
    p.n_ctx = n_ctx;
    p.n_batch = n_batch;
    p.n_gpu_layers = n_gpu_layers;
    p.seed = 1;
    p.f16_kv = false;              // Falcon always runs an f32 KV cache (examples/falcon_common.cpp:786)
    p.logits_all = logits_all != 0;
    p.embedding = embedding != 0;
    p.use_mmap = true;
    return falcon_init_from_file(path, p);
}

} // extern "C"
