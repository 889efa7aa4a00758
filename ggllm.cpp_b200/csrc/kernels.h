// kernels.h -- internal launcher declarations (C++ linkage) shared by the C ABI, the ggml_cuda_* surface and the engine.
#pragma once
#include "formats.cuh"

// ---- weights.cu
size_t wplanes_layout(WPlanes & W, int type, int K, int M);
void   wplanes_upload(WPlanes & W, int type, int K, int M, const void * host_raw, cudaStream_t stream);
void   wplanes_from_device_raw(WPlanes & W, int type, int K, int M, const void * dev_raw, cudaStream_t stream);
void   wplanes_alloc_random(WPlanes & W, int type, int K, int M, uint64_t seed, cudaStream_t stream);
void   launch_repack_rows(const WPlanes & W, const void * stage_dev, int64_t row0, int64_t nrows, cudaStream_t stream);   // raw blocks of rows [row0, row0 + nrows) -> planes
void   wplanes_free(WPlanes & W);
void   launch_dequant_rows(const WPlanes & W, const int32_t * rows_dev, int nrows, float * dst, int64_t dst_stride, cudaStream_t stream);

// ---- actquant.cu
size_t actq_bytes(int act_type, int K, int N);
void   actq_bind(ActQ & A, int act_type, int K, int N, void * base);          // carve a caller-provided buffer
void   launch_quantize_act(const float * x, int64_t x_stride, const ActQ & A, cudaStream_t stream);
void   launch_actq_to_f16(const ActQ & A, __half * dst, int64_t dst_stride, cudaStream_t stream);  // d*q -> fp16 (GEMM operand)

// ---- mmv.cu : y[n][m] = sum_k W[m][k] * xq[n][k], N small (decode), integer dots on quantised activations
enum { EPI_NONE = 0, EPI_GELU = 1, EPI_ADD2 = 2 };
struct MmvEpilogue { int kind; const float * r1; const float * r2;         // ADD2: y = (dot + r1[m]) + r2[m]
    // optional (fast kernel, N == 1, M % 256 == 0): the output row is also quantised for the NEXT mat-mul (its INIT pass,
    // ggml.c:11462-11476) by whichever CTA completes a 256-value chunk; qctr = M / 256 zero-initialised, self-resetting counters
    const ActQ * qout; unsigned * qctr;
    // The kernel in front of this one in the stream produces NOTHING this one reads, and everything it reads was complete AND flushed before
    // that kernel's main body ran (ffn_up behind qkv: both read the LayerNorm's output): with programmatic dependent launch the rows then
    // stream from the moment the CTAs are resident, and griddepcontrol.wait moves to the END of the kernel, where it only keeps the chain
    // of completions intact (whoever waits for this grid has thereby waited for the one in front of it)
    int late_wait; };
void   launch_mmv(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue epi, cudaStream_t stream);
void   launch_mmv_f(const WPlanes & W, const float * x, int64_t x_stride, int N, float * y, int64_t y_stride, cudaStream_t stream); // f16/f32 weights

// mmv_fast.cu: the tuned kernel (Q4_K, Q4_0, Q3_K); false = type / K not covered, nothing launched
bool   launch_mmv_fast(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue e, cudaStream_t stream);
struct MmvShape { int nt, j, d; };                  // NT threads per CTA, J pieces per thread, ring depth D; nt == 0: generic kernel
MmvShape mmv_fast_pick_shape(int wtype, int K);     // the shape launch_mmv_fast launches (B200_* switches included)
bool   mmv_fast_supports(int wtype, int K);
bool   mmv_fast_fills_sm(const WPlanes & W);       // its CTAs leave no registers for a side-stream kernel beside them
// ---- ops.cu
void   launch_layernorm(const float * x, int64_t x_stride, const float * g, const float * b, float * y, int64_t y_stride,
                        int n, int rows, cudaStream_t stream);              // y = norm(x)*g + b ; g,b may be null (plain ggml_norm)
// [x = (ra + rb) + x, written back] ; A1 = Q(norm(x)*g1+b1) ; A2 = Q(norm(x)*g2+b2) (optional)
void   launch_argmax(const float * x, int n, int32_t * out_a, int32_t * out_b, cudaStream_t stream);     // greedy sampling: lowest index on ties
void   launch_argmax_hist(const float * x, int n, int32_t * out, int32_t * hist, int * step, cudaStream_t stream);  // + hist[(*step)++] = id (graph-replayable)
void   launch_layernorm_q(float * x, int64_t x_stride, const float * ra, const float * rb, int64_t r_stride,
                          const float * g1, const float * b1, const ActQ * A1,
                          const float * g2, const float * b2, const ActQ * A2, int n, int rows, cudaStream_t stream);
void   launch_gelu(const float * x, float * y, int64_t n, cudaStream_t stream);
void   launch_f32_to_f16(const float * x, __half * y, int64_t n, cudaStream_t stream);     // the fp16 activation rows of an F16-weight mat-mul
void   launch_add(const float * a, const float * b, float * y, int64_t n, cudaStream_t stream);
void   launch_add3(const float * a, const float * b, const float * c, float * y, int64_t n, cudaStream_t stream);   // (a+b)+c
void   launch_mul_bcast(const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t stream);  // y[i] = a[i]*b[i%nb]
void   launch_add_bcast(const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t stream);
void   launch_scale(const float * a, float s, float * y, int64_t n, cudaStream_t stream);
struct RopeParams { int n_past; int head_dim; float theta_scale; };
float  rope_theta_scale_host(int head_dim, int n_ctx_rope, int dynamic_mode, float ntk_alpha, int freq_base);
// rotates x[t][h][head_dim] in place (token stride tok_stride, head stride head_dim), position = *n_past_dev + t (or n_past if dev ptr null)
void   launch_rope_neox(float * x, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past, const int * n_past_dev,
                        float theta_scale, cudaStream_t stream);

// ---- attention: attention.cu picks the kernel (attention_long.cu, attention_ws.cu and attention_prefill.cu hold the others)
struct AttnParams {
    int n_head, n_head_kv, head_dim;
    int n_tok;                  // new tokens (queries)
    int n_past;                 // tokens already in the cache (host value; ignored if n_past_dev != null)
    const int * n_past_dev;     // optional device scalar (CUDA-graph replay; one token)
    int n_ctx;                  // KV capacity (row count of the cache)
    int64_t qkv_stride;         // floats between consecutive tokens in the fused QKV buffer
    unsigned long long * trace; // optional timeline slot (debug)
    const ActQ * qout;          // optional: also emit the output row quantised for the wo mat-mul (its INIT pass)
    // optional fp16 shadow of this layer's cache for the prompt kernel (attention_ws.cu): k16 [n_ctx][n_head_kv][64],
    // vt16 [n_head_kv][64][attention_ctx_pad(n_ctx)] (V transposed); rope_kv_append keeps it in step with the fp32 cache
    __half * k16; __half * vt16;
    // RoPE(Q, K) with rope_theta_scale and the KV append are part of launch_attention.  fuse_rope (decode): the split-KV scores kernel
    // may do them itself, on qkv's rows in registers, instead of a kernel of their own -- qkv is then NOT rotated in place.
    int fuse_rope; float rope_theta_scale;
    // decode with n_past in a device scalar (graph replay): the caller's promise that this launch only serves contexts longer than
    // attention_long_threshold() keys, so the long-context kernels (attention_long.cu) may be captured; with a host n_past the launcher
    // decides by itself
    int long_ctx;
};
// The attention scratch starts with this many bytes of split-KV arrival counters.  Their owner zeroes them once; they re-arm themselves.
#define ATTN_CTR_BYTES 4096
int    attention_long_threshold();          // keys above which decode attention switches to attention_long.cu
// fused: rope(Q), rope(K) -> K cache append, V cache append      (libfalcon.cpp:2229-2281)
void   launch_rope_kv_append(float * qkv, float * k_cache, float * v_cache, const AttnParams & p, float theta_scale, cudaStream_t stream);
// RoPE + KV append, then out[t][h*head_dim + i] = softmax(scale * Q K^T + causal mask) V   (libfalcon.cpp:2229-2366), and p.qout.
// scratch: attention_scratch_bytes(p) bytes (null when that is 0).  Returns the number of kernels launched; folded (optional): whether
// p.qout was written by the attention kernels themselves rather than by a quantize_act of its own; rope_in_place (optional): whether
// Q and K were rotated in qkv itself (false when the split-KV kernels did RoPE in registers, p.fuse_rope).
int    launch_attention(float * qkv, float * k_cache, float * v_cache, float * out, int64_t out_stride, const AttnParams & p, float * scratch,
                        cudaStream_t stream, bool * folded = nullptr, bool * rope_in_place = nullptr);
size_t attention_scratch_bytes(const AttnParams & p);                // one token: enough for either decode tier at any position
int    attention_ctx_pad(int n_ctx);
size_t attention_shadow_halves(int n_head_kv, int n_ctx);           // halves per layer, for k16 and for vt16 each
void   launch_kv_shadow_refresh(const float * k_cache, const float * v_cache, __half * k16, __half * vt16, int n_head_kv, int n_ctx, int pos, int n, cudaStream_t stream);

// ---- gemm.cu : Y[n][m] = sum_k W[m][k] * X[n][k], N large (prompt), wgmma tensor cores
void   launch_mmq_gemm(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);

// ---- sampling.cu: falcon_main's sampling chain on the device (logit bias, repetition / frequency / presence penalties, top-k,
// tail-free, typical, top-p, temperature, mirostat 1 / 2, MT19937 draw)
#define B200_SAMPLER_MAX_WINDOW 256
#define B200_SAMPLER_MAX_BIAS 64
struct SamplerParams {
    int top_k;                          // <= 0: whole vocabulary (1..1024: block arg-max rounds, otherwise a radix sort of the row)
    float top_p; float temp; float repeat_penalty;
    float tfs_z, typical_p, frequency_penalty, presence_penalty;
    int mirostat; float mirostat_tau, mirostat_eta;
    int n_bias; int32_t bias_id[B200_SAMPLER_MAX_BIAS]; float bias_value[B200_SAMPLER_MAX_BIAS];   // unused entries zero (memcmp-comparable)
};
struct SamplerState;
SamplerState * sampler_state_alloc();
void   sampler_state_free(SamplerState * s);
size_t sampler_work_floats(int n_vocab);                       // size of launch_sample's `work` scratch
float  sampler_mu(const SamplerState * s);                     // synchronous read of the mirostat state
void   launch_sampler_init(SamplerState * s, uint32_t seed, const int32_t * window_dev, int n, int cap, float mu, cudaStream_t stream);
// tap: null, or sampler_tap_bytes(n_vocab) bytes that receive the candidate list after every stage (b200_sampler_tap)
void   launch_sample(const float * logits, int n_vocab, const SamplerParams & p, SamplerState * st, float * work, int32_t * out, int32_t * hist, int * step,
                     float * tap, cudaStream_t stream);
size_t sampler_tap_bytes(int n_vocab);
bool   sampler_tap_read(const float * tap, int n_vocab, const char * stage, const char * field, void * host, size_t bytes);

// ---- engine.cu (internal, C++ linkage): adopt a matrix that is already resident in the planar layout (no copy, not freed by the engine)
struct b200_falcon;
bool   falcon_adopt_matrix(b200_falcon * f, const char * ggcc_name, const WPlanes & W);
int    falcon_eval_begin(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, int all_logits);   // enqueue only (b200_falcon_eval's checks and return codes)
void   falcon_eval_finish(b200_falcon * f, float * logits);                                                                   // wait; logits (optional) receive what begin asked for
