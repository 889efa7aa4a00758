// ggml_surface.cu -- the reference's GPU operator surface (include/ggml_b200_cuda_surface.h == ggml-cuda.h:31-60)
// implemented on the sm_90a kernels of this library.  Linking this instead of ggml-cuda.cu makes ggml.c's executor
// (hook at ggml.c:15779-15790) and libfalcon.cpp's loader (libfalcon.cpp:1251) run unchanged.
//
// Residency model.  The reference decides per tensor: weights GPU / GPU_SPLIT (ggml_cuda_transform_tensor), graph
// nodes GPU only if ggml_cuda_assign_buffers was called with a non-zero scratch size -- which libfalcon forces to zero
// (libfalcon.cpp:1742-1745), so in practice src1 / dst of every claimed node are host tensors in the pinned compute
// buffer.  Both cases are handled: an operand with backend == GPU is used in place through its `extra`, a CPU operand
// is staged through a device scratch (H2D before, D2H after, one stream synchronize per claimed node).  The fast
// path that avoids those per-node round trips altogether is part B of ggml_b200.h (b200_falcon_*).
#include "kernels.h"
#include "ggml_abi_mirror.h"
#include "../../include/ggml_b200_cuda_surface.h"
#include "../../include/ggml_b200.h"
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace {

struct DeviceTensor {            // what tensor->extra->data_device[0] points to for tensors this backend owns
    int kind;                    // 0 = weight matrix in planar layout, 1 = plain f32 array
    WPlanes W;
    float * f32;
    size_t bytes;
};

GPUStatus g_status;              // zero-initialised; max_gpus 0 means "not limited yet"
float g_tensor_split[GGML_CUDA_MAX_DEVICES];
volatile bool g_initialized = false;
std::mutex g_init_mu;
cudaStream_t g_st = nullptr;
int g_main_device = 0;
size_t g_scratch_size = 0;       // ggml_cuda_set_scratch_size; 0 => assign_buffers is a no-op (ggml-cuda.cu:3095-3097)
uint8_t * g_scratch = nullptr; size_t g_scratch_off = 0;
DevScratch g_stage;              // staging for host-resident operands (and the mat-mul's activations)
std::mutex g_mu;                 // one claimed node at a time (only ith == 0 gets here, but evals may come from several threads)

void ensure_init() { if (!g_initialized) ggml_init_cublas(false); }

uint8_t * stage(size_t bytes) { return (uint8_t *) g_stage.get(bytes, g_st); }

inline DeviceTensor * owned(const abi::tensor * t) {
    return t->extra ? (DeviceTensor *) ((ggml_tensor_extra_gpu *) t->extra)->data_device[g_main_device] : nullptr;
}
inline bool on_gpu(const abi::tensor * t) { return t && (t->backend == abi::BACKEND_GPU || t->backend == abi::BACKEND_GPU_SPLIT); }
inline int64_t nelements(const abi::tensor * t) { return t->ne[0] * t->ne[1] * t->ne[2] * t->ne[3]; }
inline bool contiguous_f32(const abi::tensor * t) {
    return t->type == T_F32 && t->nb[0] == 4 && t->nb[1] == (size_t) t->ne[0] * 4 && t->nb[2] == t->nb[1] * t->ne[1] && t->nb[3] == t->nb[2] * t->ne[2];
}

// device pointer of an f32 operand: in place if device-resident, else staged at `slot` of the staging buffer
float * operand_in(const abi::tensor * t, uint8_t * slot) {
    if (on_gpu(t)) { DeviceTensor * d = owned(t); B200_ASSERT(d && d->kind == 1); return d->f32; }
    B200_ASSERT(contiguous_f32(t));
    B200_CUDA_CHECK(cudaMemcpyAsync(slot, t->data, (size_t) nelements(t) * 4, cudaMemcpyHostToDevice, g_st));
    return (float *) slot;
}
float * result_ptr(const abi::tensor * t, uint8_t * slot) {
    if (on_gpu(t)) { DeviceTensor * d = owned(t); B200_ASSERT(d && d->kind == 1); return d->f32; }
    B200_ASSERT(contiguous_f32(t));
    return (float *) slot;
}
void result_out(abi::tensor * t, const float * dev) {       // results must be visible where dst->backend says on return
    if (!on_gpu(t)) B200_CUDA_CHECK(cudaMemcpyAsync(t->data, dev, (size_t) nelements(t) * 4, cudaMemcpyDeviceToHost, g_st));
    B200_CUDA_CHECK(cudaStreamSynchronize(g_st));
}

void op_mul_mat(const abi::tensor * src0, const abi::tensor * src1, abi::tensor * dst) {
    DeviceTensor * w = owned(src0);
    B200_ASSERT(w && w->kind == 0 && "MUL_MAT: src0 must be a weight uploaded with ggml_cuda_transform_tensor");
    B200_ASSERT(src1->ne[2] == 1 && src1->ne[3] == 1 && src1->ne[0] == w->W.K && dst->ne[0] == w->W.M);
    const int N = (int) src1->ne[1];
    const size_t xb = round_up((size_t) N * w->W.K * 4, 256), yb = round_up((size_t) N * w->W.M * 4, 256);
    uint8_t * s = stage(xb + yb + mul_mat_scratch_bytes(w->W, N));
    const float * x = operand_in(src1, s);
    float * y = result_ptr(dst, s + xb);
    launch_mul_mat(w->W, x, w->W.K, N, y, w->W.M, EPI_NONE, s + xb + yb, g_st);             // the op b200_mul_mat runs
    dst->meta.cuda_perf_mal_mul_type = N <= MMV_MAX_N ? 1 : 16;        // device tag of --debug-timings (ggml.c:18266-18358)
    result_out(dst, y);
}

// dst = src0 (op) src1 with src1 broadcast over rows (ggml-cuda.cu:181-196: y[i % ky])
void op_binary(int op, const abi::tensor * src0, const abi::tensor * src1, abi::tensor * dst) {
    const int64_t n = nelements(src0), nb = nelements(src1);
    B200_ASSERT(nelements(dst) == n && n % nb == 0);
    uint8_t * s = stage(round_up((size_t) n * 4, 256) * 2 + round_up((size_t) nb * 4, 256));
    const float * a = operand_in(src0, s);
    const float * b = operand_in(src1, s + round_up((size_t) n * 4, 256));
    float * y = result_ptr(dst, s + round_up((size_t) n * 4, 256) + round_up((size_t) nb * 4, 256));
    if (op == abi::OP_ADD) launch_add_bcast(a, b, y, n, nb, g_st); else launch_mul_bcast(a, b, y, n, nb, g_st);
    result_out(dst, y);
}
void op_unary(int op, const abi::tensor * src0, const abi::tensor * src1, abi::tensor * dst) {
    const int64_t n = nelements(src0);
    uint8_t * s = stage(round_up((size_t) n * 4, 256) * 2);
    const float * a = operand_in(src0, s);
    float * y = result_ptr(dst, s + round_up((size_t) n * 4, 256));
    if (op == abi::OP_GELU) launch_gelu(a, y, n, g_st);
    else if (op == abi::OP_NORM) launch_layernorm(a, src0->ne[0], nullptr, nullptr, y, src0->ne[0], (int) src0->ne[0], (int) (n / src0->ne[0]), g_st);
    else if (op == abi::OP_SCALE) launch_scale(a, *(const float *) src1->data, y, n, g_st);      // scalar stays host-readable (ggml-cuda.cu:2504)
    else B200_ASSERT(!"unary op");
    result_out(dst, y);
}

// ------------------------------------------------------------------------------------------------ whole-graph takeover
// The per-node protocol above costs one H2D + D2H + stream synchronize per claimed node (241 MUL_MATs per Falcon-40B token).  The
// reference's executor, however, shows this hook EVERY node of the eval graph in execution order (ggml.c:15779-15790, 17241-17300),
// and libfalcon names its tensors (model tensors carry their GGCC names, libfalcon.cpp:1158; graph nodes "result_lm_head" etc.,
// :2116-2443).  That is enough to run the whole Falcon eval on the device-resident engine (engine.cu, part B of ggml_b200.h) behind
// the unmodified falcon_eval:
//   eval 1 ("learning", e.g. falcon_main's BOS warm-up, falcon_main.cpp:662-673) runs through the per-node path while every model
//     tensor the nodes reference is recorded by name.  At its last node the engine is built: the offloaded weight matrices are
//     ADOPTED (they already are in this library's layout, ggml_cuda_transform_tensor), the CPU-resident embedding / lm_head /
//     LayerNorm vectors are uploaded once, the KV capacity comes from "cache_k"; the engine then replays that eval to fill ITS cache.
//   eval 2.. : GET_ROWS(tok_embeddings, embd) marks the start: the token ids are on the host there.  Every node is claimed without
//     computing anything until the first ROPE node, whose src1 holds n_past and the rope context (ggml.c:6947-6952): the engine
//     evaluates the whole graph there (one CUDA graph launch for N = 1); "result_lm_head" receives the logits, and row N - 1 of
//     "result_norm" the engine's final LayerNorm row, the one row falcon_eval_internal copies for falcon_get_embeddings (:2551-2557).
//   a first eval at n_past > 0 (a session restored before it, falcon_main.cpp:662-673 then skips its BOS warm-up): the engine is built
//     the same way, imports positions [0, n_past) from the host cache that eval read (cache_k rows, V from the buffer its "V_new" view
//     wrote, column stride n_past + N) and replays the eval's N tokens at n_past.
// Conditions: every layer's four matrices offloaded (n_gpu_layers >= n_layer), head_dim 64.  Otherwise the per-node path stays in charge.
// Under takeover the reference's HOST KV cache is not maintained (the cache lives in HBM).  Session state still is what the reference
// expects: falcon_copy_state_data / falcon_set_state_data (libfalcon.cpp:4226-4470) copy the KV cache through ggml_cpy graphs over 3-D
// views of cache_k and the current V buffer, and between evals this hook serves those copies from the device cache (tk_state_copy).
// B200_NO_TAKEOVER=1 disables it.
b200_falcon * b200_takeover_engine = nullptr;          // the engine behind the hook (tests read its counters)

struct Takeover {
    enum State { OFF, LEARNING, READY, DISABLED } state = OFF;
    std::map<std::string, const abi::tensor *> named;   // GGCC name -> model tensor
    const abi::tensor * emb = nullptr, * cache_k = nullptr, * v_new = nullptr;   // v_new: the V buffer the learning eval wrote
    std::vector<int32_t> tokens; int N = 0, n_past = -1, rope_ctx = 0;
    bool active = false, launched = false;              // this eval is being evaluated by the engine
    abi::tensor * result_norm = nullptr;                // this eval's "result_norm" node, filled at "result_lm_head"
    int valid_upto = 0, n_vocab = 0, n_embd = 0, n_batch = 0;
    int n_layer = 0, n_ctx = 0, e_kv = 0;               // the engine's cache: e_kv = n_head_kv * 64 floats per position and layer
    float * logits = nullptr; size_t logits_floats = 0; // pinned
    long evals_taken = 0;                               // by this engine (the cumulative count for tests / bench is g_tk_total)
} g_tk;
long g_tk_total = 0;

// a model is being (un)loaded: whatever engine exists borrows planes of the old one
void tk_reset() {
    if (b200_takeover_engine) { b200_falcon_free(b200_takeover_engine); b200_takeover_engine = nullptr; }
    float * lg = g_tk.logits; const size_t lf = g_tk.logits_floats;
    g_tk = Takeover{};
    g_tk.logits = lg; g_tk.logits_floats = lf;
}

bool is_model_name(const char * n) { return strncmp(n, "transformer.", 12) == 0 || strcmp(n, "lm_head.weight") == 0; }
void tk_note(const abi::tensor * t) { if (t && t->name[0] && is_model_name(t->name)) g_tk.named[t->name] = t; }

const float * tk_logits(size_t floats) {
    if (floats > g_tk.logits_floats) {
        if (g_tk.logits) B200_CUDA_CHECK(cudaFreeHost(g_tk.logits));
        g_tk.logits_floats = floats; B200_CUDA_CHECK(cudaMallocHost(&g_tk.logits, floats * 4));
    }
    return g_tk.logits;
}

// end of the learning eval: build the engine from what the graph showed.  false -> stay on the per-node path for good
bool tk_build() {
    auto get = [&](const std::string & n) -> const abi::tensor * { auto it = g_tk.named.find(n); return it == g_tk.named.end() ? nullptr : it->second; };
    const abi::tensor * qkv0 = get("transformer.h.0.self_attention.query_key_value.weight"), * head = get("lm_head.weight");
    if (!qkv0 || !head || !g_tk.emb || !g_tk.cache_k) return false;
    int n_layer = 0;
    while (get("transformer.h." + std::to_string(n_layer) + ".self_attention.query_key_value.weight")) n_layer++;
    b200_falcon_params hp{};
    hp.n_embd = (int) qkv0->ne[0]; hp.n_head = hp.n_embd / 64; hp.n_head_kv = (int) ((qkv0->ne[1] / 64 - hp.n_head) / 2);
    hp.n_vocab = (int) head->ne[1]; hp.n_layer = n_layer; hp.falcon_type = get("transformer.h.0.ln_attn.weight") ? 40 : 7;
    if (hp.n_embd % 64 || hp.n_head_kv <= 0 || hp.n_head % hp.n_head_kv || (hp.n_head + 2 * hp.n_head_kv) * 64 != qkv0->ne[1]) return false;
    hp.n_ctx = (int) (nelements(g_tk.cache_k) / ((int64_t) n_layer * hp.n_head_kv * 64));
    hp.n_batch = g_tk.n_batch = 512;
    if (hp.n_ctx <= 0 || (int64_t) hp.n_ctx * n_layer * hp.n_head_kv * 64 != nelements(g_tk.cache_k)) return false;
    const char * mats[4] = { "self_attention.query_key_value.weight", "self_attention.dense.weight", "mlp.dense_h_to_4h.weight", "mlp.dense_4h_to_h.weight" };
    for (int l = 0; l < n_layer; l++)
        for (const char * m : mats) {
            const abi::tensor * t = get("transformer.h." + std::to_string(l) + "." + m);
            if (!t || !on_gpu(t) || !owned(t) || owned(t)->kind != 0) return false;                   // partial offload: keep the per-node path
        }
    b200_falcon * f = b200_falcon_create(&hp);
    B200_ASSERT(b200_falcon_set_embeddings(f, 1) == 0);        // a context with embedding = true reads "result_norm" after every eval
    bool ok = true;
    auto vec_or_mat = [&](const std::string & name) {
        const abi::tensor * t = get(name);
        if (!t) { ok = false; return; }
        if (on_gpu(t) && owned(t) && owned(t)->kind == 0) { ok = ok && falcon_adopt_matrix(f, name.c_str(), owned(t)->W); return; }
        const int64_t ne[2] = { t->ne[0], t->ne[1] };
        if (on_gpu(t) && owned(t) && owned(t)->kind == 1) {                                              // 1-D f32 that the loader offloaded (7B's input_layernorm.weight)
            std::vector<float> h((size_t) t->ne[0]);
            B200_CUDA_CHECK(cudaMemcpy(h.data(), owned(t)->f32, h.size() * 4, cudaMemcpyDeviceToHost));
            b200_falcon_set_tensor(f, name.c_str(), T_F32, 1, ne, h.data());
        } else b200_falcon_set_tensor(f, name.c_str(), t->type, t->n_dims, ne, t->data);                 // CPU-resident: one upload (mmap'ed file bytes)
    };
    vec_or_mat("transformer.word_embeddings.weight"); vec_or_mat("lm_head.weight");
    vec_or_mat("transformer.ln_f.weight"); vec_or_mat("transformer.ln_f.bias");
    for (int l = 0; l < n_layer && ok; l++) {
        const std::string p = "transformer.h." + std::to_string(l) + ".";
        for (const char * m : mats) vec_or_mat(p + m);
        if (hp.falcon_type == 40) { vec_or_mat(p + "ln_attn.weight"); vec_or_mat(p + "ln_attn.bias"); vec_or_mat(p + "ln_mlp.weight"); vec_or_mat(p + "ln_mlp.bias"); }
        else { vec_or_mat(p + "input_layernorm.weight"); vec_or_mat(p + "input_layernorm.bias"); }
    }
    if (!ok) { b200_falcon_free(f); return false; }
    b200_takeover_engine = f; g_tk.n_vocab = hp.n_vocab; g_tk.n_embd = hp.n_embd;
    g_tk.n_layer = n_layer; g_tk.n_ctx = hp.n_ctx; g_tk.e_kv = hp.n_head_kv * 64;
    return true;
}

// ---- session state behind the engine.  falcon_copy_state_data / falcon_set_state_data build, per plane, a CPY between a host blob and a
// VIEW of the host cache (E = n_head_kv * 64, n = kv_ntok, offset 0):
//   K: view of cache_k,                 ne (E, n, n_layer), nb (4, 4 E, 4 E n_ctx)  <->  blob [n_layer][n][E]
//   V: view of cache_v_a or cache_v_b,  ne (n, E, n_layer), nb (4, 4 n, 4 E n_ctx)  <->  blob [n_layer][E][n]
enum { KV_NONE, KV_K, KV_V };
int kv_view_plane(const abi::tensor * t) {
    if (!t || t->op != abi::OP_VIEW || !t->src0) return KV_NONE;
    const char * n = t->src0->name;
    if (strcmp(n, "cache_k") == 0) return KV_K;
    // cache_v: the V cache of a FALCON_NO_KV_UPGRADE build, whose layout state_view_ntok refuses
    return (strcmp(n, "cache_v_a") == 0 || strcmp(n, "cache_v_b") == 0 || strcmp(n, "cache_v") == 0) ? KV_V : KV_NONE;
}
// n if `view` has the state layout of `plane` over the engine's cache, else -1
int state_view_ntok(const abi::tensor * view, int plane) {
    const int64_t E = g_tk.e_kv, n = plane == KV_K ? view->ne[1] : view->ne[0];
    const bool dims = plane == KV_K ? view->ne[0] == E && view->nb[1] == (size_t) E * 4 : view->ne[1] == E && view->nb[1] == (size_t) n * 4;
    const bool ok = dims && view->type == T_F32 && view->data == view->src0->data && view->ne[2] == g_tk.n_layer && view->ne[3] == 1 &&
                    view->nb[0] == 4 && view->nb[2] == (size_t) E * g_tk.n_ctx * 4 && n >= 0 && n <= g_tk.n_ctx;
    return ok ? (int) n : -1;
}
// READY, no eval in flight: a CPY out of a view of the host cache is a save and is served from the device (claimed); a CPY into one is a
// restore, which the CPU performs as well, so that the host state stays what the reference expects
bool tk_state_copy(bool lead, abi::tensor * t) {
    if (t->op != abi::OP_CPY) return false;
    const int out = kv_view_plane(t->src0), in = kv_view_plane(t->src1);
    if (out == KV_NONE && in == KV_NONE) return false;
    if (!lead) return out != KV_NONE;
    const abi::tensor * view = out != KV_NONE ? t->src0 : t->src1, * host = out != KV_NONE ? t : t->src0;
    const int plane = out != KV_NONE ? out : in, n = state_view_ntok(view, plane);
    if (n < 0 || !contiguous_f32(host) || nelements(host) != nelements(view)) {
        fprintf(stderr, "b200: a copy %s the host KV cache ('%s') in a layout the device KV cache cannot serve; set B200_NO_TAKEOVER=1 to keep "
                        "the per-node path\n", out != KV_NONE ? "out of" : "into", t->name);
        abort();
    }
    const RefKvLayout L{ (size_t) n * g_tk.e_kv, (size_t) n, (size_t) n * g_tk.e_kv };
    float * blob = (float *) host->data;
    if (out != KV_NONE) {
        if (n > g_tk.valid_upto) {
            fprintf(stderr, "b200: session state of %d positions requested but the device KV cache holds %d\n", n, g_tk.valid_upto);
            abort();
        }
        if (falcon_ref_kv_export(b200_takeover_engine, n, plane == KV_K ? blob : nullptr, plane == KV_V ? blob : nullptr, L) != 0) {
            fprintf(stderr, "b200: KV state export failed (%d positions)\n", n); abort();
        }
        return true;
    }
    if (falcon_ref_kv_import(b200_takeover_engine, n, plane == KV_K ? blob : nullptr, plane == KV_V ? blob : nullptr, L) != 0) {
        fprintf(stderr, "b200: KV state import failed (%d positions)\n", n); abort();
    }
    g_tk.valid_upto = n;
    return false;
}

// returns true when the node is handled by the takeover machinery (the caller then returns true to ggml: skip the CPU)
bool tk_node(const abi::compute_params * params, abi::tensor * t) {
    if (g_tk.state == Takeover::DISABLED) return false;
    const bool lead = params->ith == 0 && params->type == abi::TASK_COMPUTE;
    const bool start = t->op == abi::OP_GET_ROWS && t->src0 && strcmp(t->src0->name, "transformer.word_embeddings.weight") == 0 && t->src1 && t->src1->type == 18 /* GGML_TYPE_I32 */;
    if (start && lead && getenv("B200_NO_TAKEOVER")) {                       // read at the start of every eval: per-node path from here on
        if (g_tk.evals_taken > 0) { fprintf(stderr, "b200: B200_NO_TAKEOVER set after the device took the KV cache over\n"); abort(); }
        g_tk.state = Takeover::OFF; g_tk.active = false;
        return false;
    }
    if (start && lead) {
        g_tk.tokens.assign((const int32_t *) t->src1->data, (const int32_t *) t->src1->data + t->src1->ne[0]);
        g_tk.N = (int) t->src1->ne[0]; g_tk.n_past = -1; g_tk.launched = false; g_tk.result_norm = nullptr;
        if (g_tk.state == Takeover::OFF) { g_tk.state = Takeover::LEARNING; g_tk.named.clear(); g_tk.emb = t->src0; }
        else if (g_tk.state == Takeover::READY) {
            if (t->src0 != g_tk.emb || g_tk.N > g_tk.n_batch) {              // another model / an oversized batch
                if (g_tk.evals_taken > 0) { fprintf(stderr, "b200: n_batch %d > %d (or a second model) behind the operator hook after the device took the KV cache over\n", g_tk.N, g_tk.n_batch); abort(); }
                g_tk.state = Takeover::DISABLED; return false;
            }
            g_tk.active = true;
        }
    }
    if (g_tk.state == Takeover::LEARNING) {
        if (lead) {
            tk_note(t->src0); tk_note(t->src1);
            if (t->op == abi::OP_ROPE && g_tk.n_past < 0) { g_tk.n_past = ((const int32_t *) t->src1->data)[0]; g_tk.rope_ctx = ((const int32_t *) t->src1->data)[3]; }
            if (t->op == abi::OP_VIEW && t->src0 && strcmp(t->src0->name, "cache_k") == 0) g_tk.cache_k = t->src0;
            if (t->op == abi::OP_VIEW && t->src0 && strcmp(t->name, "V_new") == 0) g_tk.v_new = t->src0;        // libfalcon.cpp:2264-2271
        }
        return false;                                                          // the per-node path computes this eval
    }
    if (!g_tk.active) return g_tk.state == Takeover::READY && tk_state_copy(lead, t);
    if (!lead) return true;
    if (t->op == abi::OP_ROPE && !g_tk.launched) {
        g_tk.n_past = ((const int32_t *) t->src1->data)[0]; g_tk.rope_ctx = ((const int32_t *) t->src1->data)[3];
        if (g_tk.n_past > g_tk.valid_upto) {
            fprintf(stderr, "b200: eval at n_past %d but the device KV cache holds %d positions; "
                            "set B200_NO_TAKEOVER=1 to keep the per-node path\n", g_tk.n_past, g_tk.valid_upto);
            abort();
        }
        // enqueue only: the device evaluates the graph while ggml walks (and this hook claims) the remaining nodes
        if (falcon_eval_begin(b200_takeover_engine, g_tk.tokens.data(), g_tk.N, g_tk.n_past, g_tk.rope_ctx, 1) != 0) {
            fprintf(stderr, "b200: engine eval failed behind ggml_cuda_compute_forward (N %d, n_past %d)\n", g_tk.N, g_tk.n_past); abort();
        }
        g_tk.valid_upto = g_tk.n_past + g_tk.N; g_tk.launched = true; g_tk.evals_taken++; g_tk_total++;
    }
    if (strcmp(t->name, "result_norm") == 0) g_tk.result_norm = t;
    if (strcmp(t->name, "result_lm_head") == 0) {
        B200_ASSERT(g_tk.launched && contiguous_f32(t) && nelements(t) == (int64_t) g_tk.N * g_tk.n_vocab);
        abi::tensor * rn = g_tk.result_norm;
        const int64_t E = g_tk.n_embd;
        B200_ASSERT(rn && contiguous_f32(rn) && rn->ne[0] == E && nelements(rn) == (int64_t) g_tk.N * E);
        // falcon_eval_internal reads the logits here and the last "result_norm" row for falcon_get_embeddings (libfalcon.cpp:2538-2557)
        falcon_eval_finish(b200_takeover_engine, (float *) t->data, (float *) rn->data + (size_t) (g_tk.N - 1) * E);
        t->meta.cuda_perf_mal_mul_type = g_tk.N <= MMV_MAX_N ? 1 : 16;
        g_tk.active = false;
    }
    return true;
}

// called after the per-node path has finished the LAST node of the learning eval
void tk_finish_learning() {
    if (tk_build() && g_tk.n_past >= 0 && g_tk.N <= g_tk.n_batch) {
        // positions before the eval (a restored session): the host cache this eval read, K rows and V as "V_new" left it
        const size_t lay = (size_t) g_tk.n_ctx * g_tk.e_kv;
        const bool imported = g_tk.n_past == 0 || (g_tk.v_new &&
            falcon_ref_kv_import(b200_takeover_engine, g_tk.n_past, (const float *) g_tk.cache_k->data, (const float *) g_tk.v_new->data,
                                 RefKvLayout{ lay, (size_t) (g_tk.n_past + g_tk.N), lay }) == 0);
        // replay the eval on the engine so that ITS cache holds these positions too (results discarded)
        float * lg = const_cast<float *>(tk_logits((size_t) g_tk.N * g_tk.n_vocab));
        if (imported && b200_falcon_eval(b200_takeover_engine, g_tk.tokens.data(), g_tk.N, g_tk.n_past, g_tk.rope_ctx, lg, 1) == 0) {
            g_tk.valid_upto = g_tk.n_past + g_tk.N; g_tk.state = Takeover::READY;
            if (getenv("B200_VERBOSE")) fprintf(stderr, "b200: Falcon eval graph recognised -- whole-graph evaluation on the device from the next eval on\n");
            return;
        }
    }
    if (b200_takeover_engine) { b200_falcon_free(b200_takeover_engine); b200_takeover_engine = nullptr; }
    g_tk.state = Takeover::DISABLED;                                         // until the next model load (tk_reset)
}

} // namespace

extern "C" {

// test / bench hook: number of evals the engine has run behind ggml_cuda_compute_forward (0 = per-node path only)
long b200_surface_takeover_evals(void) { return g_tk_total; }

const GPUStatus * ggml_cuda_get_system_gpu_status(void) { return &g_status; }

void ggml_cuda_update_gpu_status(int device_id) {
    (void) device_id;                                        // one device per process: -1 and 0 mean the same thing
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); count = 0; }
    if (g_main_device >= count) g_main_device = 0;
    // one process drives one GPU (see header): num_devices is 1 unless the caller forbade GPUs with max_gpus == 0 *explicitly*
    g_status.num_devices = count > 0 ? 1 : 0;
    g_status.main_device_id = 0;
    g_status.total_vram = g_status.total_free_vram = 0;
    if (g_status.num_devices) {
        int cur = 0; B200_CUDA_CHECK(cudaGetDevice(&cur));
        B200_CUDA_CHECK(cudaSetDevice(g_main_device));
        B200_CUDA_CHECK(cudaGetDeviceProperties(&g_status.device_props[0], g_main_device));
        B200_CUDA_CHECK(cudaMemGetInfo(&g_status.device_vram_free[0], &g_status.device_vram_total[0]));
        g_status.total_vram = g_status.device_vram_total[0]; g_status.total_free_vram = g_status.device_vram_free[0];
        if (cur != g_main_device) B200_CUDA_CHECK(cudaSetDevice(cur));
    }
}

bool ggml_init_cublas(bool check_only) {
    if (check_only || g_initialized) return g_initialized;
    std::lock_guard<std::mutex> lk(g_init_mu);
    if (g_initialized) return true;
    if (g_status.num_devices == 0) ggml_cuda_update_gpu_status(-1);
    if (g_status.num_devices == 0) { fprintf(stderr, "ggml_init_cublas: no CUDA device; this backend has no CPU fallback\n"); exit(1); }
    g_tensor_split[0] = 0.f;
    B200_CUDA_CHECK(cudaSetDevice(g_main_device));
    b200_init(g_main_device);
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&g_st, cudaStreamNonBlocking));
    g_initialized = true;
    return true;
}

void ggml_cuda_print_gpu_status(const GPUStatus * status, bool print_summary) {
    if (!status) { fprintf(stderr, "Error: Invalid GPU status pointer.\n"); return; }
    const char * div = "+----+------------------------------------+------------+-----------+-----------+-----------+";
    fprintf(stderr, "%s\n| ID | %-25s %2d found | %10s | %9s | %9s | %9s |\n%s\n", div, "Device", status->num_devices, "VRAM Total", "VRAM Free", "VRAM Used", "Device", div);
    for (int i = 0; i < status->num_devices; i++)
        fprintf(stderr, "| %2d | %-34s | %7zu MB | %6zu MB | %6zu MB | %9s |\n", i, status->device_props[i].name, status->device_vram_total[i] >> 20,
                status->device_vram_free[i] >> 20, (status->device_vram_total[i] - status->device_vram_free[i]) >> 20, i == status->main_device_id ? "Primary" : "Secondary");
    (void) print_summary;
    fprintf(stderr, "%s\n", div);
}

void ggml_cuda_set_max_gpus(int max_gpus) { g_status.max_gpus = max_gpus; }
void ggml_cuda_set_vram_reserved(int64_t r) { for (int i = 0; i < GGML_CUDA_MAX_DEVICES; i++) g_status.device_vram_reserved[i] = r; }
void ggml_cuda_set_tensor_split_prepare(const float * ts, int n) { for (int i = 0; i < GGML_CUDA_MAX_DEVICES; i++) g_tensor_split[i] = (ts && i < n) ? ts[i] : 0.f; }
void ggml_cuda_set_tensor_split(const float * ts) { (void) ts; /* row splits are replaced by the layer-range pipeline (ggml_b200.h part B) */ }
void ggml_cuda_set_main_device(int d) { g_main_device = d; }
void ggml_cuda_set_scratch_size(size_t s) { g_scratch_size = s; }
void ggml_cuda_free_scratch(void) { if (g_scratch) { cudaFree(g_scratch); g_scratch = nullptr; } g_scratch_off = 0; }

void * ggml_cuda_host_malloc(size_t size) { return b200_host_malloc(size); }
void ggml_cuda_host_free(void * p) { b200_host_free(p); }
void ggml_cuda_pool_reset_all_counters(int) {}                                       // no buffer pool: device memory is static
int ggml_cuda_pool_purge_buffers_with_access_count(int, int) { return 0; }

void ggml_cuda_transform_tensor(void * data, struct ggml_tensor * t_) {
    abi::tensor * t = (abi::tensor *) t_;
    ensure_init();
    if (b200_takeover_engine || g_tk.state != Takeover::OFF) tk_reset();     // a (new) model is loading
    B200_ASSERT(t->backend == abi::BACKEND_GPU || t->backend == abi::BACKEND_GPU_SPLIT);
    B200_ASSERT(t->ne[2] == 1 && t->ne[3] == 1);
    DeviceTensor * d = new DeviceTensor();
    if (t->ne[1] == 1 && t->type == T_F32) {                 // 1-D f32 (Falcon-7B's input_layernorm.weight, libfalcon.cpp:1853)
        d->kind = 1; d->bytes = (size_t) t->ne[0] * 4;
        B200_CUDA_CHECK(cudaMalloc(&d->f32, d->bytes));
        B200_CUDA_CHECK(cudaMemcpy(d->f32, data, d->bytes, cudaMemcpyHostToDevice));
    } else {
        d->kind = 0;
        wplanes_upload(d->W, t->type, (int) t->ne[0], (int) t->ne[1], data, g_st);
        d->bytes = d->W.bytes;
    }
    ggml_tensor_extra_gpu * extra = new ggml_tensor_extra_gpu();
    memset(extra, 0, sizeof(*extra));
    extra->data_device[g_main_device] = d;
    t->extra = extra;
}

void ggml_cuda_free_data(struct ggml_tensor * t_) {
    abi::tensor * t = (abi::tensor *) t_;
    if (!on_gpu(t) || !t->extra) return;
    if (b200_takeover_engine || g_tk.state != Takeover::OFF) tk_reset();     // the engine borrows these planes
    DeviceTensor * d = owned(t);
    if (d) { if (d->kind == 0) wplanes_free(d->W); else cudaFree(d->f32); delete d; }
    delete (ggml_tensor_extra_gpu *) t->extra;
    t->extra = nullptr;
}

// Graph-build-time placement of a node on the device (ggml-cuda.cu:3094-3162).  With scratch size 0 this is a no-op,
// exactly like the reference; otherwise the node gets f32 storage from a ring-allocated scratch arena (views and
// in-place results alias their source).
static void assign_impl(abi::tensor * t, bool scratch) {
    if (scratch && g_scratch_size == 0) return;
    ensure_init();
    if (t->src0 && t->src0->backend == abi::BACKEND_CPU && (t->src0->op == abi::OP_RESHAPE || t->src0->op == abi::OP_TRANSPOSE || t->src0->op == abi::OP_VIEW)) assign_impl(t->src0, scratch);
    if (t->op == abi::OP_CPY && t->src1->backend == abi::BACKEND_CPU) assign_impl(t->src1, scratch);
    t->backend = abi::BACKEND_GPU;
    DeviceTensor * d = new DeviceTensor(); d->kind = 1; d->bytes = (size_t) nelements(t) * 4;
    const bool view = t->op == abi::OP_VIEW || t->op == abi::OP_RESHAPE || t->op == abi::OP_PERMUTE || t->op == abi::OP_TRANSPOSE;
    if ((view || (t->src0 && t->data == t->src0->data)) && t->src0 && on_gpu(t->src0) && owned(t->src0)) {
        size_t off = 0;
        if (t->op == abi::OP_VIEW && t->opt[0]) memcpy(&off, t->opt[0]->data, sizeof(size_t));   // ggml-cuda.cu:3121-3124
        d->f32 = (float *) ((uint8_t *) owned(t->src0)->f32 + off);
    } else if (scratch) {
        if (!g_scratch) B200_CUDA_CHECK(cudaMalloc(&g_scratch, g_scratch_size));
        if (g_scratch_off + d->bytes > g_scratch_size) g_scratch_off = 0;
        d->f32 = (float *) (g_scratch + g_scratch_off);
        g_scratch_off += round_up(d->bytes, 256);
        B200_ASSERT(g_scratch_off <= g_scratch_size);
    } else B200_CUDA_CHECK(cudaMalloc(&d->f32, d->bytes));
    ggml_tensor_extra_gpu * extra = new ggml_tensor_extra_gpu();
    memset(extra, 0, sizeof(*extra));
    extra->data_device[g_main_device] = d;
    t->extra = extra;
}
void ggml_cuda_assign_buffers(struct ggml_tensor * t) { assign_impl((abi::tensor *) t, true); }
void ggml_cuda_assign_buffers_no_scratch(struct ggml_tensor * t) { assign_impl((abi::tensor *) t, false); }

bool ggml_cuda_can_mul_mat(const struct ggml_tensor * s0, const struct ggml_tensor * s1, struct ggml_tensor * d_) {
    const abi::tensor * src0 = (const abi::tensor *) s0, * src1 = (const abi::tensor *) s1; const abi::tensor * dst = (const abi::tensor *) d_;
    if (g_status.num_devices == 0) return false;
    if (dst->meta.cuda_op_directive != -1) return dst->meta.cuda_op_directive != 0;       // ggml-cuda.cu:2851-2853
    if (src0->meta.cuda_op_directive != -1) return src0->meta.cuda_op_directive != 0;
    if (src1->meta.cuda_op_directive != -1) return src1->meta.cuda_op_directive != 0;
    return on_gpu(src0) && src1->type == T_F32 && dst->type == T_F32;                    // never upload CPU-resident weights per call
}

void ggml_cuda_mul(const struct ggml_tensor * s0, const struct ggml_tensor * s1, struct ggml_tensor * d) {
    std::lock_guard<std::mutex> lk(g_mu);
    op_binary(abi::OP_MUL, (const abi::tensor *) s0, (const abi::tensor *) s1, (abi::tensor *) d);
}

bool ggml_cuda_compute_forward(struct ggml_compute_params * p_, struct ggml_tensor * t_) {
    const abi::compute_params * params = (const abi::compute_params *) p_;
    abi::tensor * t = (abi::tensor *) t_;
    if (t->op == abi::OP_NONE) return true;                                  // ggml-cuda.cu:3196
    if (g_status.num_devices == 0) return false;
    if (tk_node(params, t)) return true;                                     // whole-graph takeover (see above)
    const bool learning_last = g_tk.state == Takeover::LEARNING && params->ith == 0 && params->type == abi::TASK_COMPUTE && strcmp(t->name, "result_lm_head") == 0;
    struct Finish { bool on; ~Finish() { if (on) tk_finish_learning(); } } finish_after_this_node{ learning_last };
    if (t->meta.cuda_op_directive == 0) return false;                        // ggml-cuda.cu:3202 (KQ / KQV, libfalcon.cpp:2309,2356)
    const bool any_on_device = t->backend == abi::BACKEND_GPU || (t->src0 && on_gpu(t->src0)) || (t->src1 && t->src1->backend == abi::BACKEND_GPU);
    if (!any_on_device) return false;
    switch (t->op) {
        case abi::OP_MUL_MAT:
            if (!on_gpu(t->src0)) return false;
            break;
        case abi::OP_ADD: case abi::OP_MUL: case abi::OP_SCALE: case abi::OP_GELU: case abi::OP_NORM:
        case abi::OP_RESHAPE: case abi::OP_VIEW: case abi::OP_PERMUTE: case abi::OP_TRANSPOSE:
            break;
        default:
            // an operand lives on the device but the op has no device implementation behind this surface: the CPU
            // cannot read it, so fail loudly instead of computing garbage
            fprintf(stderr, "ggml_cuda_compute_forward: op %d on device-resident tensor '%s' is not supported through the per-node hook; use b200_falcon_eval\n", t->op, t->name);
            abort();
    }
    if (params->ith != 0) return true;                                       // ggml-cuda.cu:3284-3286
    if (params->type == abi::TASK_INIT || params->type == abi::TASK_FINALIZE) return true;
    ensure_init();
    std::lock_guard<std::mutex> lk(g_mu);
    switch (t->op) {
        case abi::OP_MUL_MAT: op_mul_mat(t->src0, t->src1, t); break;
        case abi::OP_ADD: case abi::OP_MUL: op_binary(t->op, t->src0, t->src1, t); break;
        case abi::OP_SCALE: case abi::OP_GELU: case abi::OP_NORM: op_unary(t->op, t->src0, t->src1, t); break;
        default: break;                                                      // views: nothing to do
    }
    return true;
}

} // extern "C"
