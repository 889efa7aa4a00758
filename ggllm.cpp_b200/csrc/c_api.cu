// c_api.cu -- part A of include/ggml_b200.h: the kernel-level C ABI.
#include "kernels.h"
#include "../../include/ggml_b200.h"
#include <mutex>
#include <cstring>
#include <vector>

struct b200_weight { WPlanes W; };
struct b200_actq { ActQ A; void * base; size_t bytes; __half * h; };

static cudaStream_t g_own_stream = nullptr;
static cudaStream_t g_stream = nullptr;
static std::mutex g_mu;

cudaStream_t b200_current_stream() { return g_stream; }
void launch_gemm_simt(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);
bool launch_gemm_tc(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);

static unsigned long long * g_trace = nullptr; static int g_trace_cap = 0, g_trace_n = 0; static char g_trace_names[4096][24];
unsigned long long * b200_trace_slot(const char * name) {
    if (!g_trace || g_trace_n >= g_trace_cap) return nullptr;
    strncpy(g_trace_names[g_trace_n], name, 23); g_trace_names[g_trace_n][23] = 0;
    return g_trace + 2 * (g_trace_n++);
}

extern "C" {

// debugging aid: per-kernel device timeline.  enable(n) allocates n slots and makes every instrumented launch claim one;
// reset() re-arms the slots (call before replaying a captured graph); dump() copies {start, end} ns pairs and names out.
void b200_trace_enable(int n_slots) {
    if (g_trace) { cudaFree(g_trace); g_trace = nullptr; }
    g_trace_cap = n_slots > 4096 ? 4096 : n_slots; g_trace_n = 0;
    if (g_trace_cap > 0) B200_CUDA_CHECK(cudaMalloc(&g_trace, (size_t) g_trace_cap * 16));
}
void b200_trace_reset(void * stream) {
    if (!g_trace) return;
    std::vector<unsigned long long> init((size_t) g_trace_cap * 2);
    for (int i = 0; i < g_trace_cap; i++) { init[2 * i] = ~0ull; init[2 * i + 1] = 0; }
    B200_CUDA_CHECK(cudaMemcpy(g_trace, init.data(), init.size() * 8, cudaMemcpyHostToDevice));
    (void) stream;
}
int b200_trace_dump(unsigned long long * out, char * names, int max_slots) {
    const int n = g_trace_n < max_slots ? g_trace_n : max_slots;
    B200_CUDA_CHECK(cudaDeviceSynchronize());
    if (n > 0) B200_CUDA_CHECK(cudaMemcpy(out, g_trace, (size_t) n * 16, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; i++) memcpy(names + 24 * i, g_trace_names[i], 24);
    return n;
}

int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int b200_init(int device) {
    std::lock_guard<std::mutex> lk(g_mu);
    B200_CUDA_CHECK(cudaSetDevice(device));
    if (!g_own_stream) {
        B200_CUDA_CHECK(cudaStreamCreateWithFlags(&g_own_stream, cudaStreamNonBlocking));
        g_stream = g_own_stream;
    }
    int sms = 0, major = 0;
    B200_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    B200_CUDA_CHECK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    if (major != 9) { fprintf(stderr, "b200: device %d has compute capability %d.x; this library is built for sm_90a (H100) only\n", device, major); exit(1); }
    return sms;
}

void b200_set_stream(void * s) { g_stream = s ? (cudaStream_t) s : g_own_stream; }
void b200_synchronize(void) { B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); }

void * b200_event_create(void) { cudaEvent_t e; B200_CUDA_CHECK(cudaEventCreate(&e)); return (void *) e; }
void b200_event_destroy(void * e) { if (e) B200_CUDA_CHECK(cudaEventDestroy((cudaEvent_t) e)); }
void b200_event_record(void * e, void * stream) { B200_CUDA_CHECK(cudaEventRecord((cudaEvent_t) e, stream ? (cudaStream_t) stream : g_stream)); }
void b200_event_synchronize(void * e) { B200_CUDA_CHECK(cudaEventSynchronize((cudaEvent_t) e)); }
float b200_event_elapsed_ms(void * a, void * b) { float ms = 0.f; B200_CUDA_CHECK(cudaEventElapsedTime(&ms, (cudaEvent_t) a, (cudaEvent_t) b)); return ms; }
void b200_stream_synchronize(void * stream) { B200_CUDA_CHECK(cudaStreamSynchronize(stream ? (cudaStream_t) stream : g_stream)); }

void * b200_malloc(size_t bytes) { void * p = nullptr; B200_CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 1)); return p; }
void b200_free(void * p) { if (p) B200_CUDA_CHECK(cudaFree(p)); }
void b200_memcpy_h2d(void * d, const void * s, size_t n) { B200_CUDA_CHECK(cudaMemcpyAsync(d, s, n, cudaMemcpyHostToDevice, g_stream)); B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); }
void b200_memcpy_d2h(void * d, const void * s, size_t n) { B200_CUDA_CHECK(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToHost, g_stream)); B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); }
void b200_memset(void * p, int v, size_t n) { B200_CUDA_CHECK(cudaMemsetAsync(p, v, n, g_stream)); }
void * b200_host_malloc(size_t bytes) {
    if (getenv("GGML_CUDA_NO_PINNED") != nullptr) return nullptr;            // ggml-cuda.cu:2080
    void * p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }   // caller falls back to pageable (ggml-cuda.cu:2088-2096)
    return p;
}
void b200_host_free(void * p) { if (p) B200_CUDA_CHECK(cudaFreeHost(p)); }

b200_weight * b200_weight_upload(int type, int64_t K, int64_t M, const void * blocks) {
    b200_weight * w = new b200_weight();
    wplanes_upload(w->W, type, (int) K, (int) M, blocks, g_stream);
    return w;
}
b200_weight * b200_weight_random(int type, int64_t K, int64_t M, uint64_t seed) {
    b200_weight * w = new b200_weight();
    wplanes_alloc_random(w->W, type, (int) K, (int) M, seed, g_stream);
    return w;
}
void b200_weight_free(b200_weight * w) { if (w) { wplanes_free(w->W); delete w; } }
size_t b200_weight_device_bytes(const b200_weight * w) { return w->W.bytes; }
void b200_dequantize_rows(const b200_weight * w, const int32_t * rows_dev, int nrows, float * dst, int64_t dst_stride) {
    launch_dequant_rows(w->W, rows_dev, nrows, dst, dst_stride, g_stream);
}

b200_actq * b200_actq_alloc(int wtype, int64_t K, int N) {
    const int at = act_type_for(wtype);
    B200_ASSERT(at >= 0);
    b200_actq * a = new b200_actq();
    a->bytes = actq_bytes(at, (int) K, N);
    B200_CUDA_CHECK(cudaMalloc(&a->base, a->bytes));
    actq_bind(a->A, at, (int) K, N, a->base);
    a->h = nullptr;
    return a;
}
b200_actq * b200_actq_alloc_f16(int wtype, int64_t K, int N) {
    b200_actq * a = b200_actq_alloc(wtype, K, N);
    B200_CUDA_CHECK(cudaMalloc(&a->h, (size_t) N * K * sizeof(__half)));
    a->A.h = a->h;
    return a;
}
void b200_actq_free(b200_actq * a) { if (a) { B200_CUDA_CHECK(cudaFree(a->base)); if (a->h) B200_CUDA_CHECK(cudaFree(a->h)); delete a; } }
void b200_actq_download_f16(const b200_actq * a, uint16_t * h) {
    B200_ASSERT(a->h);
    B200_CUDA_CHECK(cudaStreamSynchronize(g_stream));
    B200_CUDA_CHECK(cudaMemcpy(h, a->h, (size_t) a->A.N * a->A.K * sizeof(__half), cudaMemcpyDeviceToHost));
}
void b200_actq_to_f16(const b200_actq * a, void * dst, int64_t dst_stride) { launch_actq_to_f16(a->A, (__half *) dst, dst_stride, g_stream); }
void b200_quantize_act(const float * x, int64_t x_stride, b200_actq * a) { launch_quantize_act(x, x_stride, a->A, g_stream); }
void b200_actq_download(const b200_actq * a, int8_t * q, float * d, float * s, int16_t * bs) {
    const ActQ & A = a->A; const int blk = act_block(A.type);
    B200_CUDA_CHECK(cudaStreamSynchronize(g_stream));
    if (q) B200_CUDA_CHECK(cudaMemcpy(q, A.q, (size_t) A.N * A.K, cudaMemcpyDeviceToHost));
    if (d) B200_CUDA_CHECK(cudaMemcpy(d, A.d, (size_t) A.N * (A.K / blk) * 4, cudaMemcpyDeviceToHost));
    if (s && A.s) B200_CUDA_CHECK(cudaMemcpy(s, A.s, (size_t) A.N * (A.K / 32) * 4, cudaMemcpyDeviceToHost));
    if (bs) B200_CUDA_CHECK(cudaMemcpy(bs, A.bs, (size_t) A.N * (A.K / (A.type == T_Q8_K ? 16 : 32)) * 2, cudaMemcpyDeviceToHost));
}

int b200_mmv_max_n(void) { return 8; }

int b200_mmv_launch_shape(int wtype, int64_t K, int * nt_j_d) {
    const MmvShape s = mmv_fast_pick_shape(wtype, (int) K);
    if (nt_j_d) { nt_j_d[0] = s.nt; nt_j_d[1] = s.j; nt_j_d[2] = s.d; }
    return s.nt ? 1 : 0;
}

void b200_mul_mat_vec_q(const b200_weight * w, const b200_actq * a, float * y, int64_t y_stride, int epilogue, const float * r1, const float * r2) {
    MmvEpilogue e = { epilogue, r1, r2 };
    launch_mmv(w->W, a->A, y, y_stride, e, g_stream);
}

// scratch for the one-shot b200_mul_mat (quantised activations, fp16 operand); grows on demand
static void * g_scratch = nullptr; static size_t g_scratch_bytes = 0;
static void * scratch(size_t bytes) {
    if (bytes > g_scratch_bytes) {
        if (g_scratch) { B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); B200_CUDA_CHECK(cudaFree(g_scratch)); }
        g_scratch_bytes = round_up(bytes, 1 << 20);
        B200_CUDA_CHECK(cudaMalloc(&g_scratch, g_scratch_bytes));
    }
    return g_scratch;
}

void b200_mul_mat(const b200_weight * w, const float * x, int64_t x_stride, int N, float * y, int64_t y_stride) {
    const WPlanes & W = w->W;
    if (W.type == T_F32 || W.type == T_F16) { launch_mmv_f(W, x, x_stride, N, y, y_stride, g_stream); return; }
    const int at = act_type_for(W.type);
    const size_t abytes = actq_bytes(at, W.K, N);
    if (N <= b200_mmv_max_n()) {
        ActQ A; actq_bind(A, at, W.K, N, scratch(abytes));
        launch_quantize_act(x, x_stride, A, g_stream);
        MmvEpilogue e = { EPI_NONE, nullptr, nullptr };
        launch_mmv(W, A, y, y_stride, e, g_stream);
    } else {
        uint8_t * base = (uint8_t *) scratch(abytes + (size_t) N * W.K * 2);
        ActQ A; actq_bind(A, at, W.K, N, base);
        launch_quantize_act(x, x_stride, A, g_stream);
        __half * xh = (__half *) (base + abytes);
        launch_actq_to_f16(A, xh, W.K, g_stream);
        launch_mmq_gemm(W, xh, W.K, N, y, y_stride, 0, g_stream);
    }
}

int b200_mul_mat_vec_q_chain(const b200_weight * w, const b200_actq * a_in, float * y, int epilogue, b200_actq * a_out) {
    const WPlanes & W = w->W;
    if (!mmv_fast_supports(W.type, W.K) || W.M % 256 != 0 || a_in->A.N != 1 || a_out->A.K != W.M) return 0;
    if (a_out->A.type != T_Q8_K && a_out->A.type != T_Q8_0) return 0;
    static unsigned * ctr = nullptr; static int ctr_n = 0;
    if (ctr_n < W.M / 256) {
        if (ctr) { B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); B200_CUDA_CHECK(cudaFree(ctr)); }
        ctr_n = W.M / 256; B200_CUDA_CHECK(cudaMalloc(&ctr, (size_t) ctr_n * sizeof(unsigned))); B200_CUDA_CHECK(cudaMemset(ctr, 0, (size_t) ctr_n * sizeof(unsigned)));
    }
    ActQ out = a_out->A; out.N = 1;
    MmvEpilogue e = { epilogue, nullptr, nullptr, &out, ctr };
    return launch_mmv_fast(W, a_in->A, y, W.M, e, g_stream) ? 1 : 0;
}

int b200_mul_mat_f16(const b200_weight * w, const void * x_f16, int64_t x_stride, int N, float * y, int64_t y_stride, int epi_gelu, int impl) {
    if (impl == 0) { launch_gemm_simt(w->W, (const __half *) x_f16, x_stride, N, y, y_stride, epi_gelu, g_stream); return 1; }
    return launch_gemm_tc(w->W, (const __half *) x_f16, x_stride, N, y, y_stride, epi_gelu, g_stream) ? 1 : 0;
}

void b200_layernorm(const float * x, int64_t xs, const float * g, const float * b, float * y, int64_t ys, int n, int rows) { launch_layernorm(x, xs, g, b, y, ys, n, rows, g_stream); }
void b200_gelu(const float * x, float * y, int64_t n) { launch_gelu(x, y, n, g_stream); }
void b200_add(const float * a, const float * b, float * y, int64_t n) { launch_add(a, b, y, n, g_stream); }
void b200_rope_neox(float * x, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past, int n_ctx_rope, int dyn, float alpha, int freq_base) {
    launch_rope_neox(x, n_tok, n_head, head_dim, tok_stride, n_past, nullptr, rope_theta_scale_host(head_dim, n_ctx_rope, dyn, alpha, freq_base), g_stream);
}
// the attention scratch in the shared scratch block, whose bytes may hold anything: the arrival counters are zeroed on every call
static float * attention_scratch(const AttnParams & p) {
    const size_t sb = attention_scratch_bytes(p);
    if (!sb) return nullptr;
    float * sc = (float *) scratch(sb);
    B200_CUDA_CHECK(cudaMemsetAsync(sc, 0, ATTN_CTR_BYTES, g_stream));
    return sc;
}
void b200_attention(float * qkv, float * kc, float * vc, float * out, int n_head, int n_head_kv, int head_dim, int n_tok, int n_past, int n_ctx, int n_ctx_rope) {
    AttnParams p = { n_head, n_head_kv, head_dim, n_tok, n_past, nullptr, n_ctx, (int64_t) (n_head + 2 * n_head_kv) * head_dim, nullptr };
    p.rope_theta_scale = rope_theta_scale_host(head_dim, n_ctx_rope ? n_ctx_rope : n_ctx, 1, 2.0f, 0);     // libfalcon.cpp:2231-2234
    if (n_tok > 1) {
        // the warp-specialised wgmma kernel reads an fp16 shadow of the cache: built here from the caller's fp32 cache (the engine
        // keeps one up to date token by token instead); the RoPE + append kernel writes the new rows
        static __half * sh = nullptr; static size_t sh_halves = 0;
        const size_t need = head_dim == 64 ? attention_shadow_halves(n_head_kv, n_ctx) : 0;
        if (need > sh_halves) { if (sh) { B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); B200_CUDA_CHECK(cudaFree(sh)); }
            B200_CUDA_CHECK(cudaMalloc(&sh, 2 * need * sizeof(__half))); sh_halves = need; }
        if (need) {
            B200_CUDA_CHECK(cudaMemsetAsync(sh, 0, 2 * need * sizeof(__half), g_stream));
            p.k16 = sh; p.vt16 = sh + need;
            launch_kv_shadow_refresh(kc, vc, p.k16, p.vt16, n_head_kv, n_ctx, 0, n_past, g_stream);
        }
    }
    launch_attention(qkv, kc, vc, out, (int64_t) n_head * head_dim, p, attention_scratch(p), g_stream);
}

// ---- stand-alone sampler over a logits row on the device (the engine's generation loop runs the same kernel inside its step graph)
// One sampler implementation: the default-chain parameters become a chain with every extra switched off.
b200_sampling_chain sampler_chain_of(const b200_sampling_params & sp) {
    b200_sampling_chain c{};
    c.top_k = sp.top_k; c.top_p = sp.top_p; c.tfs_z = 1.0f; c.typical_p = 1.0f; c.temp = sp.temp;
    c.repeat_penalty = sp.repeat_penalty; c.frequency_penalty = 0.0f; c.presence_penalty = 0.0f; c.repeat_last_n = sp.repeat_last_n;
    c.mirostat = 0; c.mirostat_tau = 5.0f; c.mirostat_eta = 0.1f; c.seed = sp.seed; c.n_logit_bias = 0;
    return c;
}
// validates a chain (n_vocab < 0: bias ids not checked against a vocabulary yet) and converts it to the kernel's parameters
bool sampler_params_of(const b200_sampling_chain * c, int n_vocab, SamplerParams * out) {
    if (!c || c->repeat_last_n < 0 || c->repeat_last_n > B200_SAMPLER_MAX_WINDOW || c->mirostat < 0 || c->mirostat > 2) return false;
    for (float v : { c->top_p, c->tfs_z, c->typical_p, c->temp, c->repeat_penalty, c->frequency_penalty, c->presence_penalty,
                     c->mirostat_tau, c->mirostat_eta })
        if (v != v) return false;
    if (c->n_logit_bias < 0 || c->n_logit_bias > B200_SAMPLER_MAX_BIAS || (c->n_logit_bias > 0 && (!c->logit_bias_ids || !c->logit_bias_values))) return false;
    SamplerParams p;
    memset(&p, 0, sizeof(p));                                        // memcmp-comparable (the engine rebuilds its graph on a change)
    p.top_k = c->top_k; p.top_p = c->top_p; p.temp = c->temp; p.repeat_penalty = c->repeat_penalty;
    p.tfs_z = c->tfs_z; p.typical_p = c->typical_p; p.frequency_penalty = c->frequency_penalty; p.presence_penalty = c->presence_penalty;
    p.mirostat = c->mirostat; p.mirostat_tau = c->mirostat_tau; p.mirostat_eta = c->mirostat_eta;
    p.n_bias = c->n_logit_bias;
    for (int i = 0; i < p.n_bias; i++) {
        const int32_t id = c->logit_bias_ids[i];
        if (id < 0 || (n_vocab >= 0 && id >= n_vocab)) return false;
        for (int j = 0; j < i; j++) if (c->logit_bias_ids[j] == id) return false;
        if (c->logit_bias_values[i] != c->logit_bias_values[i]) return false;
        p.bias_id[i] = id; p.bias_value[i] = c->logit_bias_values[i];
    }
    *out = p;
    return true;
}
struct b200_sampler {
    SamplerState * st; SamplerParams p; float * work; size_t work_floats; int32_t * out;
    bool tap_on; float * tap; size_t tap_bytes; int tap_vocab;          // b200_sampler_tap: the arena, sized lazily like work
};
b200_sampler * b200_sampler_create_chain(const b200_sampling_chain * c, const int32_t * last_tokens, int n_last) {
    SamplerParams p;
    if (!sampler_params_of(c, -1, &p) || n_last < 0 || (n_last > 0 && !last_tokens)) return nullptr;
    b200_sampler * s = new b200_sampler();
    s->st = sampler_state_alloc(); s->p = p; s->work = nullptr; s->work_floats = 0; s->tap_on = false; s->tap = nullptr; s->tap_bytes = 0; s->tap_vocab = 0;
    B200_CUDA_CHECK(cudaMalloc(&s->out, 4));
    int32_t * w = nullptr;
    if (n_last > 0) { B200_CUDA_CHECK(cudaMalloc(&w, (size_t) n_last * 4)); B200_CUDA_CHECK(cudaMemcpyAsync(w, last_tokens, (size_t) n_last * 4, cudaMemcpyHostToDevice, g_stream)); }
    launch_sampler_init(s->st, c->seed, w, n_last, c->repeat_last_n, 2.0f * c->mirostat_tau, g_stream);
    B200_CUDA_CHECK(cudaStreamSynchronize(g_stream));
    if (w) B200_CUDA_CHECK(cudaFree(w));
    return s;
}
b200_sampler * b200_sampler_create(const b200_sampling_params * sp, const int32_t * last_tokens, int n_last) {
    if (!sp || sp->top_k < 1 || sp->top_k > 1024 || sp->repeat_last_n < 0 || sp->repeat_last_n > B200_SAMPLER_MAX_WINDOW || n_last < 0) return nullptr;
    const b200_sampling_chain c = sampler_chain_of(*sp);
    return b200_sampler_create_chain(&c, last_tokens, n_last);
}
int32_t b200_sampler_sample(b200_sampler * s, const float * logits_dev, int n_vocab) {
    if (n_vocab <= 0) return -1;
    for (int i = 0; i < s->p.n_bias; i++) if (s->p.bias_id[i] >= n_vocab) return -1;      // never written outside the row
    if (sampler_work_floats(n_vocab) > s->work_floats) {
        if (s->work) B200_CUDA_CHECK(cudaFree(s->work));
        s->work_floats = sampler_work_floats(n_vocab); B200_CUDA_CHECK(cudaMalloc(&s->work, s->work_floats * 4));
    }
    if (s->tap_on && sampler_tap_bytes(n_vocab) > s->tap_bytes) {
        if (s->tap) B200_CUDA_CHECK(cudaFree(s->tap));
        s->tap_bytes = sampler_tap_bytes(n_vocab); B200_CUDA_CHECK(cudaMalloc(&s->tap, s->tap_bytes));
    }
    s->tap_vocab = n_vocab;
    SamplerParams p = s->p;
    if (p.top_k > n_vocab) p.top_k = n_vocab;
    launch_sample(logits_dev, n_vocab, p, s->st, s->work, s->out, nullptr, nullptr, s->tap_on ? s->tap : nullptr, g_stream);
    int32_t id = -1;
    B200_CUDA_CHECK(cudaMemcpyAsync(&id, s->out, 4, cudaMemcpyDeviceToHost, g_stream));
    B200_CUDA_CHECK(cudaStreamSynchronize(g_stream));
    return id;
}
float b200_sampler_mirostat_mu(const b200_sampler * s) { B200_CUDA_CHECK(cudaStreamSynchronize(g_stream)); return sampler_mu(s->st); }
void b200_sampler_free(b200_sampler * s) { if (!s) return; sampler_state_free(s->st); cudaFree(s->work); cudaFree(s->out); cudaFree(s->tap); delete s; }
int b200_sampler_tap(b200_sampler * s, int on) {
    if (!s) return 1;
    B200_CUDA_CHECK(cudaStreamSynchronize(g_stream));
    if (!on && s->tap) { B200_CUDA_CHECK(cudaFree(s->tap)); s->tap = nullptr; s->tap_bytes = 0; }
    s->tap_on = on != 0; s->tap_vocab = 0;
    return 0;
}
int b200_sampler_tap_read(const b200_sampler * s, const char * stage, const char * field, void * host, size_t bytes) {
    if (!s || !s->tap || s->tap_vocab <= 0 || !stage || !field || !host) return 1;
    B200_CUDA_CHECK(cudaStreamSynchronize(g_stream));
    return sampler_tap_read(s->tap, s->tap_vocab, stage, field, host, bytes) ? 0 : 1;
}

// the decode step's LayerNorm node exactly as the engine launches it (cluster kernel for one row of <= 8192 values, register
// kernel otherwise): [x = (ra + rb) + x] ; a1 = Q(norm(x) * g1 + b1) ; a2 = Q(norm(x) * g2 + b2) (a2 optional)
void b200_layernorm_q(float * x, int64_t x_stride, const float * ra, const float * rb, const float * g1, const float * b1, b200_actq * a1,
                      const float * g2, const float * b2, b200_actq * a2, int n, int rows) {
    ActQ A1 = a1->A; A1.N = rows;
    ActQ A2{}; if (a2) { A2 = a2->A; A2.N = rows; }
    launch_layernorm_q(x, x_stride, ra, rb, x_stride, g1, b1, &A1, g2, b2, a2 ? &A2 : nullptr, n, rows, g_stream);
}
// the decode step's attention node as the engine launches it: RoPE + KV append, split-KV scores / values kernels, and the output row
// also quantised for the wo mat-mul -- by the attention combine step when the Q8 blocks fit the head groups (returns 1), else by
// quantize_act (returns 0); the results are the same either way
int b200_attention_decode(float * qkv, float * kc, float * vc, float * out, int n_head, int n_head_kv, int head_dim, int n_past, int n_ctx,
                          int n_ctx_rope, b200_actq * qout) {
    AttnParams p = { n_head, n_head_kv, head_dim, 1, n_past, nullptr, n_ctx, (int64_t) (n_head + 2 * n_head_kv) * head_dim, nullptr, nullptr };
    p.fuse_rope = 1; p.rope_theta_scale = rope_theta_scale_host(head_dim, n_ctx_rope ? n_ctx_rope : n_ctx, 1, 2.0f, 0);      // as the engine: RoPE + append inside
    ActQ Q{}; if (qout) { Q = qout->A; Q.N = 1; p.qout = &Q; }
    bool folded = false;
    launch_attention(qkv, kc, vc, out, (int64_t) n_head * head_dim, p, attention_scratch(p), g_stream, &folded);
    return folded ? 1 : 0;
}

} // extern "C"
