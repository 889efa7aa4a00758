/*
 * ggml_b200.h -- C ABI of libggml_b200.so, the H100 (sm_90a) quantized-inference backend for ggllm.cpp.
 *
 * Plain C: pointers, sizes and ggml type ids (enum ggml_type, ggml.h:241-262) only.  No torch / C++ types.
 * Pointers named *_dev are CUDA device pointers on the current device; everything else is host memory.
 * Errors follow the reference backend's convention (ggml-cuda.cu:22-51, ggml.h:204-210): CUDA failures print
 * to stderr and exit(1), contract violations abort(); there are no error codes to check.
 * There is NO CPU fallback: every entry point needs a CUDA device.
 *
 * Three layers are exported:
 *   1. b200_*            kernel-level operators (this file, part A): what ggml_cuda_op_* do for one graph node
 *                        (ggml-cuda.cu:2153-2518) but device-resident and with the CPU oracle's numerics.
 *   2. b200_falcon_*     the Falcon eval path (part B): loader upload + layer-range partition + falcon_eval,
 *                        i.e. the "rewired" libfalcon offload (libfalcon.cpp:1552-1959, 2011-2588, 4566).
 *   3. ggml_cuda_*       the reference's own operator surface (ggml-cuda.h:31-60), declared in
 *                        ggml_b200_cuda_surface.h, so that ggml.c / libfalcon.cpp built with -DGGML_USE_CUBLAS
 *                        link against this library unchanged.
 */
#ifndef GGML_B200_H
#define GGML_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ========================================= part A: kernel-level operators ================================= */

/* Replaces ggml_init_cublas (ggml-cuda.cu:1982-2041).  Selects `device`, creates the backend stream.
 * Returns the number of SMs.  Idempotent per device. */
int    b200_init(int device);
int    b200_device_count(void);
/* Run all subsequent b200_* work on this cudaStream_t (NULL = the backend's own stream). */
void   b200_set_stream(void * cuda_stream);
void   b200_synchronize(void);

/* CUDA-event timing on a stream (NULL = the backend stream): what bench.py times kernels with */
void * b200_event_create(void);
void   b200_event_destroy(void * ev);
void   b200_event_record(void * ev, void * cuda_stream);
void   b200_event_synchronize(void * ev);
float  b200_event_elapsed_ms(void * ev_start, void * ev_stop);
void   b200_stream_synchronize(void * cuda_stream);

/* Raw device memory helpers so that C / ctypes callers can stage buffers without another CUDA binding. */
void * b200_malloc(size_t bytes);
void   b200_free(void * p_dev);
void   b200_memcpy_h2d(void * dst_dev, const void * src, size_t bytes);
void   b200_memcpy_d2h(void * dst, const void * src_dev, size_t bytes);
void   b200_memset(void * p_dev, int value, size_t bytes);
/* pinned host memory: ggml_cuda_host_malloc / ggml_cuda_host_free (ggml-cuda.cu:2079-2103); may return NULL */
void * b200_host_malloc(size_t bytes);
void   b200_host_free(void * p);

/* ---- weights.  Replaces ggml_cuda_transform_tensor (ggml-cuda.cu:3030-3073): `blocks` is the tensor's raw
 * data exactly as stored in a GGML/GGCC file: M rows of K/blk blocks (block_q4_0 .. block_q6_K, or f16/f32 rows).
 * The device copy is re-laid out in planes (DESIGN.md "HBM layout"); the caller may free `blocks` on return. */
typedef struct b200_weight b200_weight;
b200_weight * b200_weight_upload(int ggml_type, int64_t K, int64_t M, const void * blocks);
/* well-formed pseudo-random blocks generated on the device (throughput runs on 40B/180B-sized synthetic models) */
b200_weight * b200_weight_random(int ggml_type, int64_t K, int64_t M, uint64_t seed);
void          b200_weight_free(b200_weight * w);      /* ggml_cuda_free_data, ggml-cuda.cu:3075-3092 */
size_t        b200_weight_device_bytes(const b200_weight * w);
/* dst[r][0..K) = dequantised row rows[r] (rows_dev == NULL: rows 0..nrows-1).  Bit-exact with
 * dequantize_row_q* (ggml.c:1509-1619, k_quants.c:344-877); this is ggml_get_rows (ggml.c:11975-12002). */
void          b200_dequantize_rows(const b200_weight * w, const int32_t * rows_dev, int nrows, float * dst_dev, int64_t dst_stride);

/* ---- quantised activations: the CPU mat-mul's INIT pass (ggml.c:11462-11476): rows quantised to the weight
 * type's vec_dot_type (Q8_0 / Q8_1 / Q8_K).  Codes and scales are bit-exact with the CPU on an x86 host. */
typedef struct b200_actq b200_actq;
b200_actq * b200_actq_alloc(int weight_ggml_type, int64_t K, int N);
void        b200_actq_free(b200_actq * a);
void        b200_quantize_act(const float * x_dev, int64_t x_stride, b200_actq * a);
/* test hook: copy out codes q[N*K], scales d[N*K/blk], Q8_1 sums s[N*K/32] (or NULL), block sums bs (or NULL) */
void        b200_actq_download(const b200_actq * a, int8_t * q, float * d, float * s, int16_t * bs);
/* test hooks for the prompt GEMM's fp16 operand, fp16(d * q) per value (what the GEMM path multiplies):
 * alloc_f16  : b200_actq_alloc plus an fp16 plane [N][K] that every producer writing `a` fills alongside the codes;
 * download_f16: copy that plane out as fp16 bit patterns (a must come from b200_actq_alloc_f16);
 * to_f16     : build the same operand from a's codes and scales into dst_dev [N][dst_stride] fp16 on the device. */
b200_actq * b200_actq_alloc_f16(int weight_ggml_type, int64_t K, int N);
void        b200_actq_download_f16(const b200_actq * a, uint16_t * h);
void        b200_actq_to_f16(const b200_actq * a, void * dst_dev, int64_t dst_stride);

/* ---- y[n][m] = sum_k W[m][k] x[n][k].  Replaces ggml_cuda_mul_mat (ggml-cuda.cu:2931-2951):
 * N == 1..b200_mmv_max_n(): fused dequantise + integer-dot mat-vec (replaces dequantize_mul_mat_vec*,
 *                            ggml-cuda.cu:475-845, 1121-1171)
 * larger N               : wgmma tensor-core GEMM with fused dequantisation (replaces to_fp16_cuda +
 *                            float_to_half + cublasGemmEx, ggml-cuda.cu:2353-2403)
 * x/y are fp32 device buffers with row strides in floats. */
void   b200_mul_mat(const b200_weight * w, const float * x_dev, int64_t x_stride, int N, float * y_dev, int64_t y_stride);
/* the two halves separately; epilogue: 0 none, 1 GELU (fp16-LUT semantics), 2 y = (dot + r1) + r2 */
void   b200_mul_mat_vec_q(const b200_weight * w, const b200_actq * a, float * y_dev, int64_t y_stride,
                          int epilogue, const float * r1_dev, const float * r2_dev);
/* y = epilogue(W * a_in) for N = 1 and, from the SAME kernel, a_out = Q(y): the next mat-mul's INIT-pass quantisation
 * (ggml.c:11462-11476) done chunk by chunk as the CTAs that own a 256-value chunk finish (decode: ffn_up -> ffn_down,
 * libfalcon.cpp:2389-2394).  a_out must have K == rows of w and the activation type of the next weight.
 * returns 0 if the type / shape is not covered (rows % 256 != 0, or not Q4_K / Q4_0). */
int    b200_mul_mat_vec_q_chain(const b200_weight * w, const b200_actq * a_in, float * y_dev, int epilogue, b200_actq * a_out);
/* b200_quantize_weights_rows: fp32 rows of row_len values -> weight blocks in the FILE layout on the device (Q4_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K), every block
 * of every row bit for bit what quantize_row_q*_reference (ggml.c:927-962, k_quants.c:275-843) writes when called once per row.
 * Q2_K / Q4_K / Q5_K carry their fit's codes from block to block inside a row as the reference does; block 0 of a row starts from
 * zeroed codes, where the reference reads uninitialised stack.  n_elems is a multiple of row_len.  Returns 1 on success
 * (n_elems == 0 launches nothing), 0 for a type without a device quantiser (quantise on the host then), -1 for a bad shape
 * (row_len not a positive multiple of the type's block, n_elems not a non-negative multiple of row_len). */
int    b200_quantize_weights_rows(int ggml_type, const float * x_dev, void * blocks_dev, int64_t n_elems, int64_t row_len);
/* the same with the whole buffer as one row: one call of quantize_row_q*_reference over n_elems values, as ggml_quantize_chunk makes
 * for a chunk.  Q2_K / Q4_K / Q5_K then run the buffer on one thread: quantise matrices with b200_quantize_weights_rows. */
int    b200_quantize_weights(int ggml_type, const float * x_dev, void * blocks_dev, int64_t n_elems);
/* b200_quantize_chunks: ggml_quantize_chunk (ggml.c:19479-19560) on consecutive chunks of chunk_elems values of x_dev, the last chunk
 * shorter, as falcon_quantize calls it (libfalcon.cpp:3662-3705); output in the file layout at dst_dev, bit for bit the reference's.
 * Types: F16 (F16C rounding, NaN payloads kept), Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K.  Only Q2_K / Q4_K / Q5_K
 * depend on the chunks: their fit carries codes from block to block within a chunk (zeroed at its start, where the reference reads
 * uninitialised stack), one chain per chunk; chunk_elems == n_elems is one serial chain.  hist16 (host, 16 counts, or NULL) gets the
 * reference's legacy code histograms added (the K-quants and F16 add nothing).  Synchronises when hist16 is given.  Returns the
 * bytes written, 0 for a type outside the list, -1 for a bad shape (n_elems or chunk_elems not a multiple of the type's block,
 * chunk_elems <= 0, n_elems < 0). */
int64_t b200_quantize_chunks(int ggml_type, const float * x_dev, void * dst_dev, int64_t n_elems, int64_t chunk_elems, int64_t * hist16);
int    b200_mmv_max_n(void);
/* which kernel the decode mat-vec (b200_mul_mat_vec_q / b200_mul_mat / b200_mul_mat_vec_q_chain) runs for a weight type and
 * row length K.  Returns 1 and nt_j_d = {threads per CTA, pieces per thread, ring depth} for a tuned shape; 0 (nt_j_d = {0, 0, 0})
 * when the generic ring kernel runs.  B200_MMV_GENERIC is not applied here. */
int    b200_mmv_launch_shape(int ggml_type, int64_t K, int * nt_j_d);
/* the GEMM half alone, on fp16 activations x[n][k] already on the device (what b200_mul_mat does after quantising):
 * impl 1 = wgmma tensor-core kernel (returns 0 and writes nothing if the shape is not covered: see b200_gemm_launch_shape, and x_f16_dev
 *          must be 16-byte aligned),
 * impl 0 = CUDA-core kernel with identical operand rounding (the test reference for impl 1). */
int    b200_mul_mat_f16(const b200_weight * w, const void * x_f16_dev, int64_t x_stride, int N, float * y_dev, int64_t y_stride,
                        int epilogue_gelu, int impl);
/* which kernel b200_mul_mat_f16(impl 1) runs for a weight type, M rows of K weights, N tokens x_stride halves apart and an epilogue,
 * on a 16-byte aligned x (b200_mul_mat runs the same choice on each chunk of at most 512 tokens).  Host only, no device needed.
 * Returns 1 and out = {token-tile width BN (64, 128 or 256), K split over 1 or 2 CTAs, producer} for the wgmma kernel, where the
 * producer is the weight type of a dedicated dequantiser (GGML_TYPE_Q4_K, Q4_0 or Q3_K) or -1 for the generic one; 0 (out = {0, 0, 0})
 * when the shape is not covered (N outside 1..512, K % 64 != 0, x_stride % 8 != 0) and the CUDA-core kernel runs. */
int    b200_gemm_launch_shape(int ggml_type, int64_t K, int64_t M, int N, int64_t x_stride, int epilogue_gelu, int * out);

/* ---- the other operators of the Falcon graph, CPU-oracle numerics (SURVEY.md section 9.2) */
/* y = norm(x) * g + b per row of n values (g, b may be NULL = plain ggml_norm, ggml.c:10540-10599) */
void   b200_layernorm(const float * x_dev, int64_t x_stride, const float * g_dev, const float * b_dev,
                      float * y_dev, int64_t y_stride, int n, int rows);
void   b200_gelu(const float * x_dev, float * y_dev, int64_t n);                        /* ggml.c:3461-3484 */
void   b200_add(const float * a_dev, const float * b_dev, float * y_dev, int64_t n);   /* ggml.c:8312- */
/* NeoX RoPE (mode 2) with dynamic NTK (ggml.c:12875-12898, 12957-12979) on x[n_tok][n_head][head_dim], in place */
void   b200_rope_neox(float * x_dev, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past,
                      int n_ctx_rope, int dynamic_mode, float ntk_alpha, int freq_base);
/* RoPE(Q,K) + KV append + causal multi-query attention for one layer (libfalcon.cpp:2229-2366).
 * qkv_dev: [n_tok][(n_head + 2 n_head_kv) * head_dim] (rotated in place like ggml_rope_inplace);
 * k/v cache: [n_ctx][n_head_kv][head_dim] f32; out: [n_tok][n_head * head_dim]. */
void   b200_attention(float * qkv_dev, float * k_cache_dev, float * v_cache_dev, float * out_dev,
                      int n_head, int n_head_kv, int head_dim, int n_tok, int n_past, int n_ctx, int n_ctx_rope);

/* ---- the two fused decode-step nodes exactly as the eval path launches them (per-operator parity tests at the real model widths)
 * [x = (ra + rb) + x, written back when ra != NULL] ; a1 = Q(norm(x) * g1 + b1) ; a2 = Q(norm(x) * g2 + b2) (a2 / g2 / b2 optional):
 * residual adds (libfalcon.cpp:2399-2400) + LayerNorm(s) (ggml.c:10540-10599, libfalcon.cpp:2166-2185) + the next mat-mul's INIT
 * pass (ggml.c:11462-11476).  rows == 1 and n <= 8192: thread-block-cluster kernel; otherwise one CTA per row. */
void   b200_layernorm_q(float * x_dev, int64_t x_stride, const float * ra_dev, const float * rb_dev,
                        const float * g1_dev, const float * b1_dev, b200_actq * a1,
                        const float * g2_dev, const float * b2_dev, b200_actq * a2, int n, int rows);
/* b200_attention for ONE new token with the split-KV decode kernels; qout (optional) also receives the output row quantised for
 * the wo mat-mul.  Returns 1 when that quantisation ran inside the attention combine step, 0 when it needed its own kernel. */
int    b200_attention_decode(float * qkv_dev, float * k_cache_dev, float * v_cache_dev, float * out_dev,
                             int n_head, int n_head_kv, int head_dim, int n_past, int n_ctx, int n_ctx_rope, b200_actq * qout);
/* test hooks: b200_attention / b200_attention_decode over an fp16 cache, k16 / v16 [n_ctx][n_head_kv][head_dim] fp16 bit patterns (row
 * layout, what an engine made by b200_falcon_create_kv(.., GGML_TYPE_F16) holds).  The new rows are stored rounded to fp16, and every
 * score and output reads the rounded values, the new token's own row included. */
void   b200_attention_kv16(float * qkv_dev, uint16_t * k16_dev, uint16_t * v16_dev, float * out_dev, int n_head, int n_head_kv,
                           int head_dim, int n_tok, int n_past, int n_ctx, int n_ctx_rope);
int    b200_attention_decode_kv16(float * qkv_dev, uint16_t * k16_dev, uint16_t * v16_dev, float * out_dev, int n_head, int n_head_kv,
                                  int head_dim, int n_past, int n_ctx, int n_ctx_rope, b200_actq * qout);

/* ---- sampling on the device (SURVEY 8f-2): falcon_main's chain (examples/falcon/falcon_main.cpp:896-987) over a logits row in HBM.
 * b200_sampling_params is the default chain: llama_sample_repetition_penalty over the last repeat_last_n ids, then temp <= 0 ?
 * llama_sample_token_greedy : llama_sample_top_k -> llama_sample_top_p -> llama_sample_temperature -> llama_sample_token
 * (libfalcon.cpp:3281-3307, 3433-3447, 3094-3150, 3269-3279, 3449-3468); its top_k must be 1..1024, repeat_last_n <= 256.
 * b200_sampling_chain is the whole chain, in falcon_main's order: logit bias (row[id] += value, on a copy), repetition penalty,
 * frequency and presence penalties (l -= count * frequency_penalty + (count > 0) * presence_penalty over the same window), then
 * temp <= 0 : greedy (first maximum); mirostat 1 : temperature, llama_sample_token_mirostat (m = 100, N = n_vocab of the row);
 * mirostat 2 : temperature, llama_sample_token_mirostat_v2; otherwise top-k (<= 0: whole vocabulary) -> tail-free (tfs_z) ->
 * typical (typical_p) -> top-p -> temperature -> draw.  mu starts at 2 * mirostat_tau when the sampler is created and when a
 * generate call starts (falcon_main's static mirostat_mu for one run).  1.0 switches tfs_z / typical_p / top_p / repeat_penalty
 * off, 0 the frequency / presence penalties.  Bad input is refused (NULL / 1): mirostat not 0..2, repeat_last_n outside 0..256,
 * n_logit_bias outside 0..B200_SAMPLER_MAX_BIAS, a bias id outside [0, n_vocab) or repeated, a NaN parameter.  Bias ids are
 * checked against n_vocab at every b200_sampler_sample (returns -1) and at b200_falcon_generate_chain.
 * The draw reproduces std::discrete_distribution over std::mt19937(seed), so the same seed samples the same ids as the reference,
 * except where glibc's float functions, which are not correctly rounded, move a value across a boundary (sampling.cu). */
typedef struct { int32_t top_k; float top_p; float temp; float repeat_penalty; int32_t repeat_last_n; uint32_t seed; } b200_sampling_params;
#define B200_SAMPLER_MAX_BIAS 64
typedef struct {
    int32_t top_k;                 /* <= 0: whole vocabulary */
    float   top_p, tfs_z, typical_p, temp;
    float   repeat_penalty, frequency_penalty, presence_penalty;
    int32_t repeat_last_n;         /* 0..256 */
    int32_t mirostat;              /* 0, 1, 2 */
    float   mirostat_tau, mirostat_eta;
    uint32_t seed;
    int32_t n_logit_bias;          /* 0..B200_SAMPLER_MAX_BIAS; ids unique and in [0, n_vocab); values may be -INFINITY */
    const int32_t * logit_bias_ids; const float * logit_bias_values;
} b200_sampling_chain;
typedef struct b200_sampler b200_sampler;
/* last_tokens[0..n_last): the ids already generated / in the prompt, oldest first; the last repeat_last_n of them seed the window.  NULL on bad parameters. */
b200_sampler * b200_sampler_create(const b200_sampling_params * p, const int32_t * last_tokens, int n_last);
b200_sampler * b200_sampler_create_chain(const b200_sampling_chain * p, const int32_t * last_tokens, int n_last);
int32_t        b200_sampler_sample(b200_sampler * s, const float * logits_dev, int n_vocab);   /* samples, appends the id to the window, returns it */
float          b200_sampler_mirostat_mu(const b200_sampler * s);                                /* mirostat's current mu */
void           b200_sampler_free(b200_sampler * s);
/* test hooks: the candidate list after every stage of the chain, in the order the reference's llama_sample_* functions leave it.
 * b200_sampler_tap(s, 1) makes every later b200_sampler_sample also copy its stages into a tap arena on the device (allocated at the
 * first sample, about 76 bytes per vocabulary entry); b200_sampler_tap(s, 0) frees it, and with the tap off nothing is copied.
 * b200_sampler_tap_read copies one field of the most recent sample to the host; `bytes` must be its exact size.  Stages and fields:
 *   "row"     logits [n_vocab] f32: after the logit bias and the penalties, in id order
 *   "order"   n, ids, logits: after top-k's rounds or the whole-row sort (mirostat: after the division by temp)
 *   "tfs"     n, ids, logits, p: after tail-free's cut; p is the softmax it cut on
 *   "typical" n, ids, logits, p: after typical's reordering and cut; p as above; entropy (f32)
 *   "top_p"   n, ids, logits, p: after top-p's cut
 *   "temp"    n, ids, logits: after the division by temp (default chain)
 *   "final"   n, ids, logits, p: the candidates of the draw and their probabilities; u (f64, the uniform variate; -1 when fewer
 *             than two candidates draw nothing), pick (position drawn), id, mu (after mirostat's update), k (mirostat 1's cut, else -1)
 * n, pick, id, k are int32 and the arrays hold n entries (ids int32, logits / p f32).  A stage that did not run has n = -1 and no
 * arrays.  Both return 0 on success, 1 otherwise. */
int            b200_sampler_tap(b200_sampler * s, int on);
int            b200_sampler_tap_read(const b200_sampler * s, const char * stage, const char * field, void * host, size_t bytes);

/* ---- scoring on the device: falcon_perplexity's per-token term (examples/falcon_perplexity/falcon_perplexity.cpp:12-26, 113-115).
 * For row r (logits_dev + r * row_stride, n_vocab floats) with target t = targets_dev[r]:
 *   m = max_i l[i];  e[i] = expf(l[i] - m) (float);  S = (((0.0 + e[0]) + e[1]) + ...) + e[n_vocab - 1] (double, sequential, in id order);
 *   p = (float) ((double) e[t] / S);  nll_dev[r] = -logf(p) (float; p == 0 gives +Inf).
 * expf / logf are correctly rounded (the sampler's), where glibc's differ from that in the last bit at times.  t == -1 skips the row
 * (nll_dev[r] unwritten); any other t outside [0, n_vocab) writes NaN.  Enqueued on `cuda_stream` (NULL = the backend stream). */
void           b200_token_nll(const float * logits_dev, int n_vocab, int n_rows, int64_t row_stride, const int32_t * targets_dev,
                              float * nll_dev, void * cuda_stream);

/* ========================================= part B: Falcon eval path ====================================== */

typedef struct b200_falcon b200_falcon;

typedef struct {
    int32_t n_vocab, n_embd, n_head, n_head_kv, n_layer;
    int32_t falcon_type;      /* 7 | 40: selects the single- or dual-LayerNorm layer (libfalcon.cpp:1578-1593, 2177) */
    int32_t n_ctx;            /* KV capacity (falcon_context_params.n_ctx, libfalcon.h:91) */
    int32_t n_batch;          /* largest n_tokens of one eval (libfalcon.h:92) */
    /* layer-range pipeline (replaces tensor_split / n_gpu_layers, libfalcon.h:93-97): this process owns layers
     * [layer_first, layer_last) of the model; rank/world describe its place in the NCCL pipeline. */
    int32_t layer_first, layer_last;
    int32_t rank, world;
} b200_falcon_params;

/* Create the device-resident model shell (KV cache, activation arena, CUDA graphs).  Weights are attached
 * afterwards, tensor by tensor, under the reference's GGCC tensor names (libfalcon.cpp:1764-1861), e.g.
 * "transformer.h.3.mlp.dense_h_to_4h.weight".  Tensors of layers outside [layer_first, layer_last) are ignored. */
b200_falcon * b200_falcon_create(const b200_falcon_params * params);
/* b200_falcon_create with the KV cache stored as kv_ggml_type: GGML_TYPE_F32 (0, what b200_falcon_create does) or GGML_TYPE_F16 (1,
 * falcon_context_params.f16_kv, libfalcon.h:103).  Any other type: NULL.  An fp16 cache stores K (after RoPE) and V rounded to nearest
 * even (ggml_fp32_to_fp16 on an F16C host; beyond +-65504 a value becomes +-Inf) and every attention read widens them exactly: the
 * engine computes what the f32 engine would over a cache whose rows were rounded when they were appended.  It takes half the bytes. */
b200_falcon * b200_falcon_create_kv(const b200_falcon_params * params, int kv_ggml_type);
/* b200_falcon_create_kv whose layers streamed_layers[0..n_streamed) (global indices inside [layer_first, layer_last), no repeats) keep their
 * four matrices in pinned host memory in the device's planar layout.  Each eval copies every streamed layer into one of two device
 * layer slots just before the layer runs, overlapped with the layers before it.  Results are bit for bit those of the resident engine.
 * n_streamed == 0 is b200_falcon_create_kv.  NULL for a bad layer list, a bad kv type, or world > 1. */
b200_falcon * b200_falcon_create_streamed(const b200_falcon_params * params, int kv_ggml_type, const int32_t * streamed_layers, int n_streamed);
/* number of streamed layers; layers_out (optional) gets them in ascending order.  host_bytes: the pinned images; slot_bytes: the two
 * device slots; copy_bytes: what one eval copies host -> device (the sum of the streamed layers' images).  Any pointer may be NULL. */
int           b200_falcon_stream_info(const b200_falcon * f, int32_t * layers_out, size_t * host_bytes, size_t * slot_bytes, size_t * copy_bytes);
int           b200_falcon_kv_type(const b200_falcon * f);            /* GGML_TYPE_F32 or GGML_TYPE_F16 */
size_t        b200_falcon_kv_device_bytes(const b200_falcon * f);   /* the cache plus any fp16 copy, all local layers */
void          b200_falcon_set_tensor(b200_falcon * f, const char * name, int ggml_type, int n_dims,
                                     const int64_t * ne, const void * data);
/* random-init tensor of the named shape generated on the device (synthetic throughput models) */
void          b200_falcon_set_tensor_random(b200_falcon * f, const char * name, int ggml_type, uint64_t seed);
/* load every tensor of a GGCC v10 file (format: libfalcon.cpp:770-973) through the GPU-direct path: mmap -> pinned ring buffers ->
 * cudaMemcpyAsync -> on-the-fly planar repack, several host threads, two buffers in flight each, one synchronize at the end
 * (replaces libfalcon.cpp:1196-1270 + the blocking per-tensor copy of ggml-cuda.cu:3030-3073).  The file is validated while it is
 * read (bounds, types, shapes, names); returns 0 on success, -1 on an unreadable / malformed / mismatching file. */
int           b200_falcon_load_ggcc(b200_falcon * f, const char * path);
/* seconds the last b200_falcon_load_ggcc took (header parse to the final synchronize) and the quantised-matrix bytes it streamed */
double        b200_falcon_load_seconds(const b200_falcon * f, size_t * bytes);
/* hparams of a GGCC file without loading it (fills n_vocab..falcon_type); returns 0 on success */
int           b200_ggcc_read_hparams(const char * path, b200_falcon_params * out);

/* falcon_quantize on the device: mirrors llama_model_quantize_params (libfalcon.h) */
typedef struct {
    int32_t nthread;                 /* <= 0: the host's hardware threads.  Decides the chunk plan only: see b200_quantize_ggcc */
    int32_t ftype;                   /* enum llama_ftype: 0 1 2 3 7 8 9 10 11 12 13 14 15 16 17 18 */
    int32_t allow_requantize;        /* quantised input tensors may be dequantised and quantised again */
    int32_t quantize_output_tensor;  /* 0: lm_head.weight is copied as it is (--leave-output-tensor) */
} b200_quantize_params;
typedef struct {
    uint64_t size_org, size_new;     /* tensor data bytes in and out (falcon_quantize's "model size" / "quant size") */
    int64_t  hist[16];               /* the legacy code histogram over every quantised tensor (zeros for F16 / K-quant outputs) */
    int32_t  n_tensors, n_quantized;
    double   seconds;                /* wall time, file open to file close */
    uint64_t staging_bytes;          /* size of one pinned staging buffer: a tensor is read in pieces of at most this */
    uint64_t device_bytes;           /* device memory the pipeline allocated */
} b200_quantize_report;
/* b200_quantize_ggcc: falcon_model_quantize (libfalcon.cpp:3533-3743) with the quantisers on the device: the output file is byte for
 * byte the reference's.  A tensor is quantised iff its name ends in "weight", it is 2-D, it is not lm_head.weight when
 * quantize_output_tensor is 0, and its type differs from the ftype's; every other tensor is copied.  F16 and quantised inputs are
 * widened / dequantised on the device exactly as the reference converts them.  Chunk plan: nthread_use = nthread > 1 ?
 * min(nthread, ceil(n / 16384)) : 1; with nthread_use < 2 a tensor is ONE chunk, otherwise chunks of 16384 values -- for Q2_K / Q4_K /
 * Q5_K a single chunk is one serial chain over the whole tensor (slow for large tensors, and what the reference defines).
 * Pipeline: the input is mapped; each tensor goes through pinned staging buffers (report->staging_bytes each) to the device, is
 * converted, quantised and copied back while the host reads the next tensor and writes the previous one.  Device memory: two input
 * buffers of the largest quantised tensor as stored, one fp32 buffer and one output buffer of it (about 10 bytes per value of the
 * largest tensor for an F16 input).  The input is untrusted and bounds-checked as b200_falcon_load_ggcc checks it.  report may be
 * NULL.  Returns 0 on success, 1 where the reference refuses (unknown ftype, a K-quant output for a tensor whose ne[0] is not a
 * multiple of 256, a quantised input without allow_requantize; the output file is then not written), -1 for an unreadable or
 * malformed input or an I/O error. */
int           b200_quantize_ggcc(const char * path_in, const char * path_out, const b200_quantize_params * params, b200_quantize_report * report);
void          b200_falcon_free(b200_falcon * f);
size_t        b200_falcon_weight_bytes(const b200_falcon * f);   /* algorithmic bytes of the quantised matrices, streamed layers' included */

/* NCCL pipeline plumbing (world > 1): rank 0 creates the id, every rank passes the same 128 bytes. */
void          b200_nccl_unique_id(void * id128);
void          b200_falcon_init_pipeline(b200_falcon * f, const void * id128);

/* falcon_eval (libfalcon.cpp:4566): n_tokens token ids at position n_past.  Host buffers in and out:
 * token ids H2D and logits D2H are part of the call.  logits: n_vocab floats of the last token, or
 * n_tokens * n_vocab if all_logits (falcon_context_params.logits_all).  n_ctx_rope = the rope's 4th parameter
 * (n_max_real_ctx ? that : n_ctx, libfalcon.cpp:2229-2230); 0 = use n_ctx.
 * In a pipeline every rank calls it; only the last rank's `logits` are written.  Returns 0 on success. */
int           b200_falcon_eval(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope,
                               float * logits, int all_logits);
/* falcon_context_params.embedding (libfalcon.h:108): with it on, every b200_falcon_eval also brings the last token's row of the final
 * LayerNorm ("result_norm", libfalcon.cpp:2422-2431) to the host, in the same synchronise as its logits; the row is exactly the fp32
 * values the head quantises for lm_head.  Off by default, and off changes nothing.  Returns 0, or 1 on a rank without the head. */
int           b200_falcon_set_embeddings(b200_falcon * f, int on);
/* falcon_get_embeddings (libfalcon.h:267): n_embd floats, the row of the most recent b200_falcon_eval; NULL with embeddings off, before
 * any eval and after any other eval call (b200_falcon_score / _perplexity / _decode_dev / _generate*, which do not produce it).  The
 * buffer is the engine's and is overwritten by the next eval. */
const float * b200_falcon_embeddings(const b200_falcon * f);
/* b200_falcon_eval that scores its rows on the device instead of returning logits (single GPU): targets[i] in [0, n_vocab) scores
 * row i -- nll[i] (host) receives b200_token_nll's term for it -- and -1 skips it (nll[i] untouched).  No logits cross PCIe.
 * A batch with a scored row runs the final LayerNorm and lm_head over all n_tokens rows, exactly as b200_falcon_eval(all_logits = 1)
 * does, so the scored logits are bit for bit that call's; a batch without one runs no head.  One token replays the decode step graph.
 * Returns b200_falcon_eval's codes (0, 1, 2), 3 for a target outside [-1, n_vocab) (checked before anything runs), 1 on a pipeline
 * engine (world > 1) or a NULL nll with a scored row. */
int           b200_falcon_score(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope,
                                const int32_t * targets, float * nll);
/* falcon_perplexity (examples/falcon_perplexity/falcon_perplexity.cpp:28-123) over tokens[0, n_tokens): n_chunk = n_tokens / n_ctx
 * chunks (the tail is dropped); chunk c evaluates tokens[c n_ctx, (c + 1) n_ctx) in batches of the engine's n_batch at n_past
 * 0, n_batch, ... with the rope context n_ctx and no BOS substitution, and scores rows k in [min(512, n_ctx / 2), n_ctx - 1) against
 * tokens[c n_ctx + k + 1] through b200_falcon_score.  The terms are summed in double in k order over all chunks so far and
 * ppl[c] = exp(sum / count) after chunk c (what the reference prints as [c+1]).  nll (optional) receives the terms, n_chunk *
 * (n_ctx - 1 - min(512, n_ctx / 2)) floats; ppl (optional) n_chunk doubles.  The tokens go H2D once and only the terms come back.
 * Returns n_chunk (>= 0), or -1 for n_ctx < 2, n_ctx above the engine's n_ctx, a token outside the vocabulary or world > 1. */
int           b200_falcon_perplexity(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_ctx, double * ppl, float * nll);
/* device-resident decode step for throughput measurement: token id already on the device, logits stay on the
 * device (b200_falcon_logits_dev).  Same kernels/graph as b200_falcon_eval minus the two PCIe copies. */
int           b200_falcon_decode_dev(b200_falcon * f, const int32_t * token_dev, int n_past, int n_ctx_rope);   /* 0 = ok, 1 = n_past outside [0, n_ctx) */
const float * b200_falcon_logits_dev(const b200_falcon * f);
/* greedy generation without leaving the device (single GPU): feeds `first_token` at position n_past, then n_steps times
 * "decode, arg-max of the logits (lowest index on ties), use it as the next token".  tokens_out[i] = token sampled after
 * step i.  What falcon_main does with top_k = 1 (llama_sample_token_greedy, libfalcon.cpp:3464-3473), minus the 260 KB
 * logits D2H and the host scan per token (SURVEY 8f-2).  Returns 0 on success. */
int           b200_falcon_generate_greedy(b200_falcon * f, int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out);
/* KV cache rows [pos, pos + n) of one (global) layer index, host buffers of n * n_head_kv * head_dim floats each (either may be NULL).
 * The host rows are f32 for either cache type: an fp16 cache is widened exactly by kv_read and rounded to nearest even by kv_write.
 * The building block of session save / restore (falcon_copy_state_data / falcon_set_state_data, libfalcon.cpp:4313-4490) over the
 * device-resident cache.  Return 0 on success, 1 if the layer is not on this rank or the range leaves [0, n_ctx). */
int           b200_falcon_kv_read(b200_falcon * f, int layer, int pos, int n, float * k_out, float * v_out);
int           b200_falcon_kv_write(b200_falcon * f, int layer, int pos, int n, const float * k_in, const float * v_in);
/* the fp16 copy of the cache that prompt chunks of more than b200_mmv_max_n() tokens attend over (kept only when n_batch exceeds it;
 * in an fp16 engine k16_out is the K cache itself, always there, and vt16_out only when n_batch exceeds it):
 * positions [pos, pos + n) of one layer as fp16 bit patterns, k16_out [n][n_head_kv][head_dim] and vt16_out [n_head_kv][head_dim][n]
 * (V transposed; either may be NULL).  The range may extend past n_ctx to n_ctx rounded up to 64, the padding of the transposed copy.
 * Return 0 on success, 1 if the engine keeps no such copy, the layer is not on this rank or the range is invalid. */
int           b200_falcon_kv_shadow_read(b200_falcon * f, int layer, int pos, int n, uint16_t * k16_out, uint16_t * vt16_out);
/* session file over the device KV cache (what falcon_save_session_file / falcon_load_session_file keep of the KV state,
 * libfalcon.cpp:4490-4563), in this library's own container: positions [0, n_tokens) of every local layer.  save: 0 / -1.
 * load: the number of positions restored (continue evaluating at that n_past), -1 on a missing / truncated / mismatching file. */
int           b200_falcon_save_kv(b200_falcon * f, const char * path, int n_tokens);
int           b200_falcon_load_kv(b200_falcon * f, const char * path);
/* pseudo-random K / V rows for positions [pos, pos + n) of every local layer, generated on the device (long-context throughput runs;
 * an fp16 cache holds the same values rounded) */
int           b200_falcon_kv_fill_random(b200_falcon * f, int pos, int n, uint64_t seed);
/* b200_falcon_generate_greedy with the sampling chain above run on the device after every step (every rank of a pipeline calls it with
 * the same arguments; the last rank samples).  Returns 0 on success, 1 on bad arguments. */
int           b200_falcon_generate(b200_falcon * f, const b200_sampling_params * p, const int32_t * last_tokens, int n_last,
                                   int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out);
/* the same with the whole chain (b200_sampling_chain above); mu and the penalty window persist across the steps of one call */
int           b200_falcon_generate_chain(b200_falcon * f, const b200_sampling_chain * p, const int32_t * last_tokens, int n_last,
                                         int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out);
/* the cudaStream_t the eval path runs on (for event timing) */
void *        b200_falcon_stream(b200_falcon * f);
/* roofline probe: every quantised mat-vec of this rank's resident layers (4 per layer; streamed layers are left out, their matrices
 * are in HBM only while an eval runs them) + lm_head launched back to back,
 * `reps` passes, timed with CUDA events on the eval stream.  Returns total ms; fills the launch count and the
 * algorithmic weight bytes streamed in that region. */
float         b200_falcon_profile_matvec(b200_falcon * f, int reps, int * n_launches, size_t * bytes);
/* test hooks: the engine's intermediates.  b200_falcon_tap(f, 1) (after the tensors are set) allocates a tap arena with one slice per
 * local layer, sized for n_batch tokens; while it is on, every eval (eager or captured decode graph) also enqueues device-to-device
 * copies of its buffers into it on the eval stream: at the end of each layer, after both branches are complete and before the next
 * layer's LayerNorm overwrites anything, and once after the head.  b200_falcon_tap(f, 0) frees it; with the tap off nothing is enqueued.
 * Either call drops the captured decode graphs (they hold the copies).
 * b200_falcon_tap_read copies one tapped buffer of the most recent eval to the host; `bytes` must be its exact size.
 *   layer = a local (global index) layer, nodes at its end:
 *     "inp" the layer's input residual [N][n_embd] f32; "qkv" [N][(n_head + 2 n_head_kv) head_dim] f32 (RoPE applied in place or not,
 *     see "qkv_rotated"); "att", "ao", "dn" [N][n_embd] f32; "up" [N][4 n_embd] f32 (after GELU);
 *     quantised activations "xa", "xm", "xatt", "xup" (fused paths) as "<name>.q" int8 codes [N][K], ".d" f32 scales [N][K/blk],
 *     ".s" f32 Q8_1 sums [N][K/32], ".bs" int16 block sums (b200_actq_download's layout);
 *     prompt GEMM path: fp16 operand planes "xh_m" (xm's), "xh_b" (xup's), "xh_a" (xatt's at that point) [N][K];
 *     generic path: "gen_na", "gen_nm" the fp32 LayerNorm outputs [N][n_embd];
 *     "qkv_rotated" one int: 1 if RoPE rotated Q and K inside qkv, 0 if the attention kernels rotated them in registers.
 *   layer = -1 (last rank), after the head: "inp" the final residual [N][n_embd]; "xf.*" (quantised head) or "gen_na" (generic head) and
 *     "logits", each over the head's rows (the last one, or all N with all_logits).
 * Returns 0, or non-zero for a tap that is off, an unknown node, a layer that is not local or not tapped, or a wrong size.
 * b200_falcon_tap_layers(f, layers, n) switches the tap on for the n listed (global index) layers only: a slice each plus the head's,
 * so a prompt batch of a deep model can be checked a few layers at a time (one Falcon-40B slice at n_batch 512 is about 234 MB).
 * Returns non-zero, with the tap off, for a layer that is not local or listed twice. */
int           b200_falcon_tap(b200_falcon * f, int on);
int           b200_falcon_tap_layers(b200_falcon * f, const int * layers, int n);
int           b200_falcon_tap_read(const b200_falcon * f, int layer, const char * node, void * host, size_t bytes);
/* number of kernel launches (graph nodes) issued by the most recent eval on this rank; a streamed layer's copies are not counted */
int           b200_falcon_last_launches(const b200_falcon * f);
int           b200_attention_long_launches(void);     /* diagnostics: launches (eager or captured) of the long-context decode attention kernels so far */
/* CUDA-event time (ms) of the most recent eval's device work on this rank */
float         b200_falcon_last_ms(const b200_falcon * f);

#ifdef __cplusplus
}
#endif
#endif /* GGML_B200_H */
