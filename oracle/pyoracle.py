"""ctypes bindings for the oracle (TEST INFRASTRUCTURE ONLY).

Two checkers live behind this module:

* ``orc``  -- oracle/libggml_oracle.so, our own plain-C restatement of the reference's hot path
  (oracle/ggml_oracle.c; always buildable, travels to the GPU box as source + .so).
* ``ref``  -- oracle/_ref/libggml_ref.so and libfalcon_ref.so: the UNMODIFIED reference compiled from
  /root/reference by oracle/Makefile (only buildable where /root/reference exists; the prebuilt .so files
  travel to the GPU box).  Used to pin ``orc`` and as the CPU baseline.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
The product (ggllm.cpp_b200/) never does.
"""
import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# enum ggml_type (ggml.h:241-262)
F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q8_1, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, Q8_K = 0, 1, 2, 3, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15
TYPE_NAMES = {F32: "f32", F16: "f16", Q4_0: "q4_0", Q4_1: "q4_1", Q5_0: "q5_0", Q5_1: "q5_1", Q8_0: "q8_0", Q8_1: "q8_1",
              Q2_K: "q2_K", Q3_K: "q3_K", Q4_K: "q4_K", Q5_K: "q5_K", Q6_K: "q6_K", Q8_K: "q8_K"}
WEIGHT_TYPES = [Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K]
BLOCK_ELEMS = {F32: 1, F16: 1, Q4_0: 32, Q4_1: 32, Q5_0: 32, Q5_1: 32, Q8_0: 32, Q8_1: 32,
               Q2_K: 256, Q3_K: 256, Q4_K: 256, Q5_K: 256, Q6_K: 256, Q8_K: 256}
BLOCK_BYTES = {F32: 4, F16: 2, Q4_0: 18, Q4_1: 20, Q5_0: 22, Q5_1: 24, Q8_0: 34, Q8_1: 40,
               Q2_K: 84, Q3_K: 110, Q4_K: 144, Q5_K: 176, Q6_K: 210, Q8_K: 292}
VEC_DOT_TYPE = {Q4_0: Q8_0, Q5_0: Q8_0, Q8_0: Q8_0, Q4_1: Q8_1, Q5_1: Q8_1, Q2_K: Q8_K, Q3_K: Q8_K, Q4_K: Q8_K, Q5_K: Q8_K, Q6_K: Q8_K}


def row_bytes(t, k):
    assert k % BLOCK_ELEMS[t] == 0
    return k // BLOCK_ELEMS[t] * BLOCK_BYTES[t]


def _fp(a):
    return a.ctypes.data_as(C.c_void_p)


def build(ref=None):
    """Compile the C restatement (always) and oracle/_ref (when /root/reference is present)."""
    subprocess.check_call(["make", "-s", "-C", HERE, "all"])
    if ref is None:
        ref = os.path.isdir("/root/reference")
    if ref:
        subprocess.check_call(["make", "-s", "-C", HERE, "ref"])


# ----------------------------------------------------------------------------------------------- orc
class _Orc:
    def __init__(self):
        path = os.path.join(HERE, "libggml_oracle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = self.L = C.CDLL(path)
        L.orc_f32_to_f16.restype = C.c_uint16
        L.orc_f32_to_f16.argtypes = [C.c_float]
        L.orc_f16_to_f32.restype = C.c_float
        L.orc_f16_to_f32.argtypes = [C.c_uint16]
        L.orc_quantize_row.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_quantize_row_fresh_codes.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_dequantize_row.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_quantize_row_q8_0_x86.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_quantize_row_q8_1_x86.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_vec_dot.restype = C.c_float
        L.orc_vec_dot.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_void_p]
        L.orc_mul_mat.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int]
        L.orc_norm.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_layernorm.argtypes = [C.c_void_p] * 4 + [C.c_int64]
        L.orc_gelu.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_soft_max.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_rope_neox.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int]
        L.orc_rope_theta_scale.restype = C.c_float
        L.orc_rope_theta_scale.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_int]
        L.orc_falcon_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
        L.orc_falcon_eval_range.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                            C.c_int, C.c_int, C.c_void_p, C.c_void_p]

    def quantize(self, t, x, fresh_codes=False):
        """x: float32 [..., k] -> uint8 [..., row_bytes] (quantize_row_q*_reference, row by row).  fresh_codes: start every
        block's make_qkx1_quants from zeroed codes instead of the previous block's (orc_quantize_row_fresh_codes)."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.shape[-1]
        out = np.zeros(x.shape[:-1] + (row_bytes(t, k),), dtype=np.uint8)
        x2, o2 = x.reshape(-1, k), out.reshape(-1, out.shape[-1])
        fn = self.L.orc_quantize_row_fresh_codes if fresh_codes else self.L.orc_quantize_row
        for r in range(x2.shape[0]):
            assert fn(t, _fp(x2[r]), _fp(o2[r]), k) == 0
        return out

    def quantize_act(self, wtype, x):
        """activation rows -> the vec_dot_type of `wtype`, as an x86 host quantises them in mul_mat."""
        at = VEC_DOT_TYPE[wtype]
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.shape[-1]
        out = np.zeros(x.shape[:-1] + (row_bytes(at, k),), dtype=np.uint8)
        x2, o2 = x.reshape(-1, k), out.reshape(-1, out.shape[-1])
        for r in range(x2.shape[0]):
            if at == Q8_0:
                self.L.orc_quantize_row_q8_0_x86(_fp(x2[r]), _fp(o2[r]), k)
            elif at == Q8_1:
                self.L.orc_quantize_row_q8_1_x86(_fp(x2[r]), _fp(o2[r]), k)
            else:
                self.L.orc_quantize_row(Q8_K, _fp(x2[r]), _fp(o2[r]), k)
        return out

    def dequantize(self, t, q, k):
        q = np.ascontiguousarray(q, dtype=np.uint8)
        rb = row_bytes(t, k)
        out = np.zeros(q.shape[:-1] + (k,), dtype=np.float32)
        q2, o2 = q.reshape(-1, rb), out.reshape(-1, k)
        for r in range(q2.shape[0]):
            assert self.L.orc_dequantize_row(t, _fp(q2[r]), _fp(o2[r]), k) == 0
        return out

    def vec_dot(self, wt, k, w, aq):
        return float(self.L.orc_vec_dot(wt, k, _fp(np.ascontiguousarray(w)), _fp(np.ascontiguousarray(aq))))

    def mul_mat(self, wt, W, K, M, X, nthreads=8):
        """W: raw bytes of M rows; X: float32 [N][K] -> Y float32 [N][M] (ggml_compute_forward_mul_mat_q_f32)."""
        X = np.ascontiguousarray(X, dtype=np.float32).reshape(-1, K)
        W = np.ascontiguousarray(W)
        Y = np.zeros((X.shape[0], M), dtype=np.float32)
        self.L.orc_mul_mat(wt, _fp(W), K, M, _fp(X), X.shape[0], _fp(Y), nthreads)
        return Y

    def norm(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        for r in range(x.reshape(-1, x.shape[-1]).shape[0]):
            self.L.orc_norm(_fp(x.reshape(-1, x.shape[-1])[r]), _fp(y.reshape(-1, x.shape[-1])[r]), x.shape[-1])
        return y

    def layernorm(self, x, g, b):
        x = np.ascontiguousarray(x, dtype=np.float32)
        g = np.ascontiguousarray(g, dtype=np.float32)
        b = np.ascontiguousarray(b, dtype=np.float32)
        y = np.empty_like(x)
        x2, y2 = x.reshape(-1, x.shape[-1]), y.reshape(-1, x.shape[-1])
        for r in range(x2.shape[0]):
            self.L.orc_layernorm(_fp(x2[r]), _fp(g), _fp(b), _fp(y2[r]), x.shape[-1])
        return y

    def gelu(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        self.L.orc_gelu(_fp(x), _fp(y), x.size)
        return y

    def soft_max(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        x2, y2 = x.reshape(-1, x.shape[-1]), y.reshape(-1, x.shape[-1])
        for r in range(x2.shape[0]):
            self.L.orc_soft_max(_fp(x2[r]), _fp(y2[r]), x.shape[-1])
        return y

    def rope_neox(self, x, n_past, n_ctx_rope, dynamic=1, alpha=2.0, freq_base=0):
        """x: float32 [n_tok][n_head][head_dim] contiguous; returns rotated copy."""
        y = np.array(x, dtype=np.float32, order="C", copy=True)
        n_tok, n_head, hd = y.shape
        self.L.orc_rope_neox(_fp(y), n_tok, n_head, hd, n_head * hd, n_past, n_ctx_rope, dynamic, alpha, freq_base)
        return y

    def theta_scale(self, head_dim, n_ctx_rope, dynamic=1, alpha=2.0, freq_base=0):
        return float(self.L.orc_rope_theta_scale(head_dim, n_ctx_rope, dynamic, alpha, freq_base))


class _OrcTensor(C.Structure):
    _fields_ = [("type", C.c_int), ("ne0", C.c_int64), ("ne1", C.c_int64), ("data", C.c_void_p)]


class _OrcLayer(C.Structure):
    _fields_ = [(n, _OrcTensor) for n in ("ln_attn_g", "ln_attn_b", "ln_mlp_g", "ln_mlp_b", "wqkv", "wo", "ffn_up", "ffn_down")]


class _OrcModel(C.Structure):
    _fields_ = [("n_vocab", C.c_int), ("n_embd", C.c_int), ("n_head", C.c_int), ("n_head_kv", C.c_int), ("n_layer", C.c_int),
                ("falcon_type", C.c_int), ("n_ctx", C.c_int),
                ("tok_embeddings", _OrcTensor), ("ln_f_g", _OrcTensor), ("ln_f_b", _OrcTensor), ("lm_head", _OrcTensor),
                ("layers", C.POINTER(_OrcLayer)), ("k_cache", C.c_void_p), ("v_cache", C.c_void_p)]


class OrcFalcon:
    """orc_falcon_eval over a model given as {tensor name: (ggml type, shape ne, raw uint8/float32 ndarray)}
    (the dict ggllm_cpp_b200.ggcc.read_ggcc returns) -- restatement of falcon_eval_internal."""

    def __init__(self, hparams, tensors, n_ctx):
        self.orc = orc()
        self.hp = hparams
        self.keep = []
        m = self.m = _OrcModel()
        m.n_vocab, m.n_embd, m.n_head, m.n_head_kv = hparams["n_vocab"], hparams["n_embd"], hparams["n_head"], hparams["n_head_kv"]
        m.n_layer, m.falcon_type, m.n_ctx = hparams["n_layer"], hparams["falcon_type"], n_ctx

        def T(name):
            t, ne, arr = tensors[name]
            arr = np.ascontiguousarray(arr)
            self.keep.append(arr)
            return _OrcTensor(t, ne[0], ne[1] if len(ne) > 1 else 1, arr.ctypes.data)

        m.tok_embeddings, m.lm_head = T("transformer.word_embeddings.weight"), T("lm_head.weight")
        m.ln_f_g, m.ln_f_b = T("transformer.ln_f.weight"), T("transformer.ln_f.bias")
        self.layers = (_OrcLayer * m.n_layer)()
        for i in range(m.n_layer):
            p = "transformer.h.%d." % i
            L = self.layers[i]
            if m.falcon_type == 40:
                L.ln_attn_g, L.ln_attn_b = T(p + "ln_attn.weight"), T(p + "ln_attn.bias")
                L.ln_mlp_g, L.ln_mlp_b = T(p + "ln_mlp.weight"), T(p + "ln_mlp.bias")
            else:
                L.ln_mlp_g, L.ln_mlp_b = T(p + "input_layernorm.weight"), T(p + "input_layernorm.bias")
            L.wqkv, L.wo = T(p + "self_attention.query_key_value.weight"), T(p + "self_attention.dense.weight")
            L.ffn_up, L.ffn_down = T(p + "mlp.dense_h_to_4h.weight"), T(p + "mlp.dense_4h_to_h.weight")
        m.layers = C.cast(self.layers, C.POINTER(_OrcLayer))
        hd = m.n_embd // m.n_head
        self.k = np.zeros((m.n_layer, n_ctx, m.n_head_kv * hd), dtype=np.float32)
        self.v = np.zeros_like(self.k)
        m.k_cache, m.v_cache = self.k.ctypes.data, self.v.ctypes.data

    def eval(self, tokens, n_past, n_ctx_rope=None, all_logits=False, nthreads=8):
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        n = tokens.size
        out = np.zeros((n if all_logits else 1, self.m.n_vocab), dtype=np.float32)
        rc = self.orc.L.orc_falcon_eval(C.byref(self.m), _fp(tokens), n, n_past, n_ctx_rope or self.m.n_ctx, _fp(out), int(all_logits), nthreads)
        assert rc == 0
        return out

    def eval_range(self, tokens, n_past, layer_first, layer_last, resid_in=None, n_ctx_rope=None, all_logits=False, nthreads=8):
        """one pipeline stage: returns the residual stream [N][n_embd] if layer_last < n_layer, else the logits"""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        n = tokens.size
        is_last = layer_last >= self.m.n_layer
        out = np.zeros((n if all_logits else 1, self.m.n_vocab), dtype=np.float32)
        resid = np.zeros((n, self.m.n_embd), dtype=np.float32)
        rin = np.ascontiguousarray(resid_in, dtype=np.float32) if resid_in is not None else None
        rc = self.orc.L.orc_falcon_eval_range(C.byref(self.m), _fp(tokens), n, n_past, n_ctx_rope or self.m.n_ctx, _fp(out), int(all_logits),
                                              nthreads, layer_first, layer_last, _fp(rin) if rin is not None else None, _fp(resid))
        assert rc == 0
        return out if is_last else resid


# ----------------------------------------------------------------------------------------------- ref
class _QuantizeFns(C.Structure):   # quantize_fns_t, ggml.h:1585-1592
    _fields_ = [("dequantize_row_q", C.c_void_p), ("quantize_row_q", C.c_void_p), ("quantize_row_q_reference", C.c_void_p),
                ("quantize_row_q_dot", C.c_void_p), ("vec_dot_q", C.c_void_p), ("vec_dot_type", C.c_int)]


_DEQ = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int)
_QNT = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int)
_DOT = C.CFUNCTYPE(None, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p)


class _Ref:
    """The unmodified reference's codec table: ggml_internal_get_quantize_fn (ggml.h:1594)."""

    def __init__(self):
        self.L = C.CDLL(os.path.join(HERE, "_ref", "libggml_ref.so"))
        # the legacy codecs read fp16 through table_f32_f16, which only ggml_init fills (ggml.c:4277-4295)
        class _InitParams(C.Structure):
            _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]
        self.L.ggml_init.restype = C.c_void_p
        self.L.ggml_init.argtypes = [_InitParams]
        self.L.ggml_free.argtypes = [C.c_void_p]
        self.L.ggml_free(self.L.ggml_init(_InitParams(1 << 20, None, False)))
        self.L.ggml_internal_get_quantize_fn.restype = _QuantizeFns
        self.L.ggml_internal_get_quantize_fn.argtypes = [C.c_size_t]
        self.fns = {}
        for t in WEIGHT_TYPES + [Q8_1, Q8_K]:
            f = self.L.ggml_internal_get_quantize_fn(t)
            self.fns[t] = dict(deq=_DEQ(f.dequantize_row_q) if f.dequantize_row_q else None,
                               qnt=_QNT(f.quantize_row_q) if f.quantize_row_q else None,
                               qref=_QNT(f.quantize_row_q_reference) if f.quantize_row_q_reference else None,
                               qdot=_QNT(f.quantize_row_q_dot) if f.quantize_row_q_dot else None,
                               dot=_DOT(f.vec_dot_q) if f.vec_dot_q else None, vdt=f.vec_dot_type)
        # Q8_K has no table entry of its own; it is an exported symbol (k_quants.c:899-949)
        q8k = C.cast(self.L.quantize_row_q8_K_reference, _QNT)
        self.fns[Q8_K] = dict(deq=C.cast(self.L.dequantize_row_q8_K, _DEQ), qnt=q8k, qref=q8k, qdot=q8k, dot=None, vdt=Q8_K)

    def quantize(self, t, x, which="qref"):
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.shape[-1]
        out = np.zeros(x.shape[:-1] + (row_bytes(t, k),), dtype=np.uint8)
        x2, o2 = x.reshape(-1, k), out.reshape(-1, out.shape[-1])
        for r in range(x2.shape[0]):
            (self.fns[t][which] or self.fns[t]["qnt"])(_fp(x2[r]), _fp(o2[r]), k)
        return out

    def quantize_act(self, wtype, x):
        """quantize_row_q_dot of the weight type: exactly what mul_mat's INIT pass calls (ggml.c:11462-11476)."""
        at = VEC_DOT_TYPE[wtype]
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.shape[-1]
        out = np.zeros(x.shape[:-1] + (row_bytes(at, k),), dtype=np.uint8)
        x2, o2 = x.reshape(-1, k), out.reshape(-1, out.shape[-1])
        for r in range(x2.shape[0]):
            self.fns[wtype]["qdot"](_fp(x2[r]), _fp(o2[r]), k)
        return out

    def dequantize(self, t, q, k):
        q = np.ascontiguousarray(q, dtype=np.uint8)
        rb = row_bytes(t, k)
        out = np.zeros(q.shape[:-1] + (k,), dtype=np.float32)
        q2, o2 = q.reshape(-1, rb), out.reshape(-1, k)
        for r in range(q2.shape[0]):
            self.fns[t]["deq"](_fp(q2[r]), _fp(o2[r]), k)
        return out

    def vec_dot(self, wt, k, w, aq):
        s = C.c_float(0)
        self.fns[wt]["dot"](k, C.addressof(s), _fp(np.ascontiguousarray(w)), _fp(np.ascontiguousarray(aq)))
        return float(s.value)


class RefFalcon:
    """The unmodified reference's falcon_eval through oracle/ref_harness.cpp (CPU build, or the
    -DGGML_USE_CUBLAS 'hook' build whose ggml_cuda_* symbols our libggml_b200.so provides)."""

    def __init__(self, path, n_ctx, n_batch=512, logits_all=False, hook=False, n_gpu_layers=0):
        name = "libfalcon_hook.so" if hook else "libfalcon_ref.so"
        self.L = C.CDLL(os.path.join(HERE, "_ref", name), mode=C.RTLD_GLOBAL if False else C.DEFAULT_MODE)
        self.L.refh_load.restype = C.c_void_p
        self.L.refh_load.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int]
        self.L.refh_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        self.L.refh_n_vocab.argtypes = [C.c_void_p]
        self.L.refh_free.argtypes = [C.c_void_p]
        self.L.refh_print_timings.argtypes = [C.c_void_p]
        self.logits_all = logits_all
        self.h = self.L.refh_load(path.encode(), n_ctx, n_batch, n_gpu_layers, int(logits_all))
        if not self.h:
            raise RuntimeError("reference failed to load " + path)
        self.n_vocab = self.L.refh_n_vocab(self.h)

    def eval(self, tokens, n_past, n_threads=8, n_max_real_ctx=0):
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        out = np.zeros((tokens.size if self.logits_all else 1, self.n_vocab), dtype=np.float32)
        rc = self.L.refh_eval(self.h, _fp(tokens), tokens.size, n_past, n_threads, n_max_real_ctx, _fp(out), int(self.logits_all))
        assert rc == 0
        return out

    def set_seed(self, seed):
        self.L.refh_set_seed.argtypes = [C.c_void_p, C.c_int]
        self.L.refh_set_seed(self.h, seed)

    def sample(self, logits, last_tokens, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1):
        """falcon_main's default sampling chain (the reference's own llama_sample_* functions) on one logits row"""
        self.L.refh_sample.restype = C.c_int
        self.L.refh_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
        lg = np.ascontiguousarray(logits, dtype=np.float32)
        lt = np.ascontiguousarray(last_tokens, dtype=np.int32)
        return int(self.L.refh_sample(self.h, _fp(lg), lg.size, _fp(lt), lt.size, top_k, top_p, temp, repeat_penalty))

    def close(self):
        if self.h:
            self.L.refh_free(self.h)
            self.h = None


def ref_quantize_file(src, dst, ftype, nthread=8):
    """falcon_model_quantize (libfalcon.cpp:3914) via the harness; ftype = enum llama_ftype (libfalcon.h:112-131)."""
    L = C.CDLL(os.path.join(HERE, "_ref", "libfalcon_ref.so"))
    L.refh_quantize.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    rc = L.refh_quantize(src.encode(), dst.encode(), ftype, nthread)
    assert rc == 0
    return dst


_orc = None
_ref = None


def orc():
    global _orc
    if _orc is None:
        _orc = _Orc()
    return _orc


def have_ref():
    return os.path.exists(os.path.join(HERE, "_ref", "libggml_ref.so"))


def have_ref_falcon():
    return os.path.exists(os.path.join(HERE, "_ref", "libfalcon_ref.so"))


def ref():
    global _ref
    if _ref is None:
        _ref = _Ref()
    return _ref


def synth_vector(n, offset=0.0):
    """the generator of the reference's own codec test: x[i] = 0.1 + 2*cosf(i + offset) (tests/test-quantize-fns.cpp:26-30)"""
    i = np.arange(n, dtype=np.float32)
    return (np.float32(0.1) + np.float32(2.0) * np.cos(i + np.float32(offset), dtype=np.float32)).astype(np.float32)
