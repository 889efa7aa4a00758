"""The final LayerNorm row that falcon_get_embeddings returns (libfalcon.cpp:2409-2435, copied for the last token at :2551-2557), from
the unmodified reference and from the oracle's restatement, and DESIGN §2's bounds applied to it.

RefEmbedding is pyoracle.RefFalcon over a context loaded with falcon_context_params.embedding = true (oracle/ref_embedding.cpp, built
by oracle/embedding.mk); the row is read with the reference's own falcon_get_embeddings through ctypes."""
import ctypes as C
import os
import struct
import numpy as np
import pyoracle as po

EMB_CPU = os.path.join(po.HERE, "_ref", "libfalcon_emb.so")
EMB_HOOK = os.path.join(po.HERE, "_ref", "libfalcon_hook_emb.so")


class RefEmbedding(po.RefFalcon):
    def __init__(self, path, n_ctx, n_batch=512, logits_all=False, hook=False, n_gpu_layers=0, embedding=True):
        self.L = C.CDLL(EMB_HOOK if hook else EMB_CPU)
        self.L.refh_load_ex.restype = C.c_void_p
        self.L.refh_load_ex.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        self.L.refh_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        self.L.refh_n_vocab.argtypes = [C.c_void_p]
        self.L.refh_free.argtypes = [C.c_void_p]
        self.L.falcon_n_embd.argtypes = [C.c_void_p]
        self.L.falcon_get_embeddings.restype = C.POINTER(C.c_float)
        self.L.falcon_get_embeddings.argtypes = [C.c_void_p]
        self.L.llama_save_session_file.restype = C.c_bool
        self.L.llama_save_session_file.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        self.logits_all = logits_all
        self.h = self.L.refh_load_ex(path.encode(), n_ctx, n_batch, n_gpu_layers, int(logits_all), int(embedding))
        if not self.h:
            raise RuntimeError("reference failed to load " + path)
        self.n_vocab = self.L.refh_n_vocab(self.h)
        self.n_embd = self.L.falcon_n_embd(self.h)

    def embeddings(self):
        """a copy of falcon_get_embeddings: n_embd floats of the most recent falcon_eval"""
        return np.ctypeslib.as_array(self.L.falcon_get_embeddings(self.h), (self.n_embd,)).copy()

    def save_session(self, path, tokens):
        t = np.ascontiguousarray(tokens, np.int32)
        assert self.L.llama_save_session_file(self.h, str(path).encode(), t.ctypes.data, t.size)


def session_embedding(path):
    """the embedding section of a session file (llama_save_session_file -> falcon_copy_state_data, libfalcon.cpp:4226-4267)"""
    b = open(path, "rb").read()
    assert struct.unpack_from("<II", b, 0) == (0x6767736E, 1)
    o = 8 + 9 * 4                                             # falcon_hparams: eight int32 and the ftype enum
    o += 4 + 4 * struct.unpack_from("<I", b, o)[0]            # the tokens
    o += 8 + 64 * 1024                                        # rng: size and LLAMA_MAX_RNG_STATE bytes
    cap = struct.unpack_from("<Q", b, o)[0]; o += 16 + 4 * cap  # logits: capacity, size, capacity floats
    n = struct.unpack_from("<Q", b, o)[0]
    return np.frombuffer(b, np.float32, n, o + 8).copy()


def orc_embedding(o, tensors, tokens, n_past, n_ctx_rope=None):
    """orc_falcon_eval's final LayerNorm row of the last token, the KV cache advanced as by OrcFalcon.eval.  orc_falcon_eval_range
    returns the residual stream instead of running the head when layer_last < n_layer, so the layers run with n_layer one higher."""
    n_layer = o.m.n_layer
    o.m.n_layer = n_layer + 1
    try:
        resid = o.eval_range(tokens, n_past, 0, n_layer, n_ctx_rope=n_ctx_rope)
    finally:
        o.m.n_layer = n_layer
    return po.orc().layernorm(resid[-1:], tensors["transformer.ln_f.weight"][2], tensors["transformer.ln_f.bias"][2])[0]


def loose_and_tight(got, want, gemm=False):
    """DESIGN §2 with S = max|want|: asserts the loose bound (the prompt GEMM path's with gemm) and returns whether the tight one holds"""
    S = float(np.abs(want).max())
    d = np.abs(np.asarray(got, np.float32) - want)
    mx, md = (3e-2, 5e-3) if gemm else (2e-2, 2e-3)
    assert d.max() <= mx * S and np.median(d) <= md * S, (float(d.max()), float(np.median(d)), S)
    return bool(np.median(d) <= 2e-5 * S)
