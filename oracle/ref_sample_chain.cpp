// ref_sample_chain.cpp -- falcon_main's whole sampling chain (examples/falcon/falcon_main.cpp:896-987) over a caller-provided
// logits row, through the UNMODIFIED reference's public llama_sample_* functions only.
//
// TEST INFRASTRUCTURE ONLY.  Built by oracle/sample_chain.mk into oracle/_ref/libfalcon_chain.so together with the reference
// objects that `make -C oracle ref` compiled (CPU build).  The context handle comes from refh_load (ref_harness.cpp, linked in);
// its n_vocab is what mirostat 1 uses as N, and its std::mt19937 drives every draw (reseed with refh_set_seed).
#include "libfalcon.h"
#include <vector>

extern "C" {

// top_k <= 0: the whole row (falcon_main.cpp:858).  logit bias: row[id] += value (falcon_main.cpp:899-902) on a private copy.
// mu: in/out state of mirostat 1 / 2 (falcon_main keeps it in a static that starts at 2 * tau).
int refh_sample_chain(void * h, const float * logits, int n_vocab, const int * last_tokens, int n_last,
                      int top_k, float top_p, float tfs_z, float typical_p, float temp,
                      float repeat_penalty, float frequency_penalty, float presence_penalty,
                      int mirostat, float mirostat_tau, float mirostat_eta, float * mu,
                      int n_bias, const int * bias_ids, const float * bias_values) {
    falcon_context * ctx = (falcon_context *) h;
    std::vector<float> row(logits, logits + n_vocab);
    for (int i = 0; i < n_bias; i++) row[bias_ids[i]] += bias_values[i];
    std::vector<falcon_token_data> candidates;
    candidates.reserve(n_vocab);
    for (falcon_token id = 0; id < n_vocab; id++) candidates.emplace_back(falcon_token_data{ id, row[id], 0.0f });
    falcon_token_data_array cp = { candidates.data(), candidates.size(), false };
    llama_sample_repetition_penalty(ctx, &cp, last_tokens, (size_t) n_last, repeat_penalty);
    llama_sample_frequency_and_presence_penalties(ctx, &cp, last_tokens, (size_t) n_last, frequency_penalty, presence_penalty);
    if (temp <= 0) return llama_sample_token_greedy(ctx, &cp);
    if (mirostat == 1) {
        llama_sample_temperature(ctx, &cp, temp);
        return llama_sample_token_mirostat(ctx, &cp, mirostat_tau, mirostat_eta, 100, mu);
    }
    if (mirostat == 2) {
        llama_sample_temperature(ctx, &cp, temp);
        return llama_sample_token_mirostat_v2(ctx, &cp, mirostat_tau, mirostat_eta, mu);
    }
    llama_sample_top_k(ctx, &cp, top_k <= 0 ? n_vocab : top_k, 1);
    llama_sample_tail_free(ctx, &cp, tfs_z, 1);
    llama_sample_typical(ctx, &cp, typical_p, 1);
    llama_sample_top_p(ctx, &cp, top_p, 1);
    llama_sample_temperature(ctx, &cp, temp);
    return llama_sample_token(ctx, &cp);
}

} // extern "C"
