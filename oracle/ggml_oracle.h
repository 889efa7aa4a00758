/*
 * ggml_oracle.h -- CPU restatement of the reference's quantized-inference hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (ggllm.cpp_b200/, include/) may include, link or
 * call this; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline/reference legs do, and only
 * as the checker.  Every function cites the reference file:line (under /root/reference) it restates.
 *
 * Parity pinning: tests/test_oracle_vs_reference.py checks every function below against the UNMODIFIED
 * reference compiled into oracle/_ref/ (bit-exact for codecs, fp tolerance for dots/evals), against the
 * committed golden vectors in tests/golden/ (made by tests/golden/make_golden.py from oracle/_ref), and
 * against the acceptance thresholds of the reference's own tests/test-quantize-fns.cpp:18-30.
 */
#ifndef GGML_ORACLE_H
#define GGML_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* tensor type ids == enum ggml_type (ggml.h:241-262) */
enum orc_type {
    ORC_F32 = 0, ORC_F16 = 1, ORC_Q4_0 = 2, ORC_Q4_1 = 3, ORC_Q5_0 = 6, ORC_Q5_1 = 7, ORC_Q8_0 = 8, ORC_Q8_1 = 9,
    ORC_Q2_K = 10, ORC_Q3_K = 11, ORC_Q4_K = 12, ORC_Q5_K = 13, ORC_Q6_K = 14, ORC_Q8_K = 15,
};

/* fp16 <-> fp32, round-to-nearest-even like F16C (ggml.c:370-395 GGML_COMPUTE_FP32_TO_FP16) */
uint16_t orc_f32_to_f16(float f);
float    orc_f16_to_f32(uint16_t h);

/* elements / bytes per block of a type (ggml.c:3625-3670 GGML_BLCK_SIZE / GGML_TYPE_SIZE); 0 if unknown */
int    orc_block_elems(int type);
size_t orc_block_bytes(int type);
size_t orc_row_bytes(int type, int64_t k);
/* activation type a weight type is dotted with (quantize_fns[].vec_dot_type, ggml.c:1627-1718) */
int    orc_vec_dot_type(int type);

/* weight codecs.  k = number of elements, multiple of the block size.  Return 0 on success, -1 bad type.
 * quantize  : quantize_row_q*_reference (ggml.c:927-1129, 1292-1325; k_quants.c:275,396,542,652,781,899)
 * dequantize: dequantize_row_q*         (ggml.c:1509-1619; k_quants.c:344,472,607,734,845,936)          */
int orc_quantize_row(int type, const float *x, void *y, int64_t k);
/* orc_quantize_row with make_qkx1_quants's code buffer zeroed at every block (Q2_K, Q4_K, Q5_K; other types as
 * orc_quantize_row).  orc_quantize_row carries the codes from block to block as the reference does (k_quants.c:275, 542,
 * 652 declare L once per row); this variant computes every block on its own, so a case where the two differ is one where
 * a quantiser that drops the carried codes would be wrong. */
int orc_quantize_row_fresh_codes(int type, const float *x, void *y, int64_t k);
int orc_dequantize_row(int type, const void *x, float *y, int64_t k);

/* Q8_0 / Q8_1 activation quantisation as the x86 host executes it: the AVX/AVX2 bodies of
 * quantize_row_q8_0 / quantize_row_q8_1 (ggml.c:1201-1237, 1421-1500): id = 127/amax,
 * q = round-half-even(x*id).  (orc_quantize_row(ORC_Q8_0..) is the scalar *_reference with roundf.) */
void orc_quantize_row_q8_0_x86(const float *x, void *y, int64_t k);
void orc_quantize_row_q8_1_x86(const float *x, void *y, int64_t k);

/* dot product of one quantised weight row with one quantised activation row, scalar order
 * (ggml.c:2591-2609, 2716-2733, 2952-2974, 3208-3230, 3321-3333; k_quants.c:1267-1305, 1684-1745,
 * 1999-2055, 2340-2400, 2748-2789).  `aq` must be of orc_vec_dot_type(wtype). */
float orc_vec_dot(int wtype, int64_t k, const void *w, const void *aq);

/* Y[n][m] = sum_k W[m][k] * X[n][k]: ggml_compute_forward_mul_mat_q_f32 (ggml.c:11318-11529):
 * X rows quantised to vec_dot_type (x86 flavour for Q8_0/Q8_1), then vec_dot per (row, column).
 * For ORC_F32 / ORC_F16 weights: plain fp32 dot (ggml.c:10911-11102 / 11104-11316 semantics,
 * F16: activations rounded to fp16 first, ggml.c:11232-11251).  nthreads>1 splits rows. */
void orc_mul_mat(int wtype, const void *W, int64_t K, int64_t M, const float *X, int64_t N, float *Y, int nthreads);

/* non-matmul ops of the Falcon graph (SURVEY.md section 9.2) */
void orc_norm(const float *x, float *y, int64_t n);                          /* ggml.c:10568-10595, eps 1e-5 */
void orc_layernorm(const float *x, const float *g, const float *b, float *y, int64_t n); /* + libfalcon.cpp:2166-2185 */
void orc_gelu(const float *x, float *y, int64_t n);                          /* ggml.c:3461-3484 fp16 LUT */
void orc_soft_max(const float *x, float *y, int64_t n);                      /* ggml.c:12427-12449 */
/* NeoX rope (mode 2) with dynamic NTK: ggml.c:12875-12898, 12957-12979.  x: [n_tok][n_head][head_dim] with
 * token stride `tok_stride` floats; rotated in place; position of token t = n_past + t. */
void orc_rope_neox(float *x, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past, int n_ctx_rope,
                   int dynamic_mode, float ntk_alpha, int freq_base);
float orc_rope_theta_scale(int head_dim, int n_ctx_rope, int dynamic_mode, float ntk_alpha, int freq_base);

/* ---- whole-model restatement: falcon_eval_internal (libfalcon.cpp:2011-2588) ---- */
typedef struct {
    int type;           /* orc_type of the data */
    int64_t ne0, ne1;   /* ne0 = contiguous (K), ne1 = rows (M); 1-D tensors: ne1 = 1 */
    const void *data;
} orc_tensor;

typedef struct {
    orc_tensor ln_attn_g, ln_attn_b;   /* 40B only: transformer.h.N.ln_attn.{weight,bias}            */
    orc_tensor ln_mlp_g,  ln_mlp_b;    /* 40B: ln_mlp.*  ; 7B: input_layernorm.*  (libfalcon.cpp:1847-1855) */
    orc_tensor wqkv, wo, ffn_up, ffn_down;
} orc_layer;

typedef struct {
    int n_vocab, n_embd, n_head, n_head_kv, n_layer, falcon_type /* 7 | 40 */;
    int n_ctx;          /* KV capacity */
    orc_tensor tok_embeddings, ln_f_g, ln_f_b, lm_head;
    orc_layer *layers;
    /* KV cache: K [n_layer][n_ctx][n_head_kv*head_dim], V same logical content (the reference keeps V
     * transposed and ping-ponged, libfalcon.cpp:2256-2281; values are identical) */
    float *k_cache, *v_cache;
} orc_model;

/* logits: [N][n_vocab] if all_logits else [n_vocab] of the last token.  n_ctx_rope = the 4th rope parameter
 * (configuration.n_max_real_ctx ? that : n_ctx, libfalcon.cpp:2229-2230).  Returns 0 on success. */
int orc_falcon_eval(orc_model *m, const int32_t *tokens, int N, int n_past, int n_ctx_rope,
                    float *logits, int all_logits, int nthreads);
/* layers [layer_first, layer_last) only: residual in (layer_first > 0) / residual out (layer_last < n_layer) */
int orc_falcon_eval_range(orc_model *m, const int32_t *tokens, int N, int n_past, int n_ctx_rope,
                          float *logits, int all_logits, int nthreads, int layer_first, int layer_last,
                          const float *resid_in, float *resid_out);

#ifdef __cplusplus
}
#endif
#endif
