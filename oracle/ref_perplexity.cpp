// ref_perplexity.cpp -- the reference's falcon_perplexity softmax (examples/falcon_perplexity/falcon_perplexity.cpp:12-26) for ctypes.
//
// TEST INFRASTRUCTURE ONLY.  Built by oracle/perplexity.mk into oracle/_ref/libfalcon_ppl.so together with the reference's
// falcon_perplexity.cpp compiled in place; no arithmetic of its own.
#include <vector>

std::vector<float> softmax(const std::vector<float> & logits);     // falcon_perplexity.cpp

extern "C" {

// softmax(row[0..n))[target], the probability falcon_perplexity.cpp:113 takes the log of
float refh_ppl_prob(const float * row, int n, int target) {
    const std::vector<float> l(row, row + n);
    return softmax(l)[target];
}

} // extern "C"
