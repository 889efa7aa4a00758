"""The oracle's falcon_eval (oracle/ggml_oracle.c, orc_falcon_eval) restated over the oracle's own operators, with a choice of KV cache:
kv_f16=False is orc_falcon_eval itself, bit for bit (tests/test_kv16.py holds it to that); kv_f16=True rounds every K / V row to fp16
as it is stored -- a ggml_cpy into an F16 cache -- so that every read, the current token's own row included, sees the rounded value.
That is the twin of an engine made by b200_falcon_create_kv(.., GGML_TYPE_F16).

The matrices, LayerNorms, GELU, RoPE and softmax are the oracle's C functions; only the attention dot products and the KV store are
written here, in float32 with the C loop's order (the oracle is built with -ffp-contract=off: one rounding per operation)."""
import numpy as np


class Kv16Twin:
    def __init__(self, orc, hparams, tensors, n_ctx, kv_f16):
        self.orc, self.hp, self.t, self.n_ctx, self.kv_f16 = orc, dict(hparams), tensors, n_ctx, kv_f16
        hd = hparams["n_embd"] // hparams["n_head"]
        self.k = np.zeros((hparams["n_layer"], n_ctx, hparams["n_head_kv"] * hd), np.float32)
        self.v = np.zeros_like(self.k)

    def _mm(self, name, X):
        t, ne, arr = self.t[name]
        return self.orc.mul_mat(t, arr, ne[0], ne[1], X)

    def _vec(self, name):
        return np.ascontiguousarray(self.t[name][2], np.float32)

    def eval(self, tokens, n_past, all_logits=False):
        hp, o = self.hp, self.orc
        E, H, HKV = hp["n_embd"], hp["n_head"], hp["n_head_kv"]
        D, G = E // H, H // HKV
        tokens = np.asarray(tokens, np.int32)
        N, T = tokens.size, n_past + tokens.size
        assert T <= self.n_ctx
        et, ene, earr = self.t["transformer.word_embeddings.weight"]
        raw = np.ascontiguousarray(earr).view(np.uint8).reshape(ene[1], -1)
        inp = o.dequantize(et, raw[tokens], ene[0])                                              # ggml_get_rows
        scale = np.float32(1.0) / np.sqrt(np.float32(D))
        for il in range(hp["n_layer"]):
            p = "transformer.h.%d." % il
            if hp["falcon_type"] == 40:
                xm = o.layernorm(inp, self._vec(p + "ln_mlp.weight"), self._vec(p + "ln_mlp.bias"))
                xa = o.layernorm(inp, self._vec(p + "ln_attn.weight"), self._vec(p + "ln_attn.bias"))
            else:
                xm = xa = o.layernorm(inp, self._vec(p + "input_layernorm.weight"), self._vec(p + "input_layernorm.bias"))
            qkv = self._mm(p + "self_attention.query_key_value.weight", xa)
            q = o.rope_neox(qkv[:, :H * D].reshape(N, H, D), n_past, self.n_ctx)
            k = o.rope_neox(qkv[:, H * D:(H + HKV) * D].reshape(N, HKV, D), n_past, self.n_ctx)
            v = qkv[:, (H + HKV) * D:]
            if self.kv_f16:
                k, v = k.astype(np.float16).astype(np.float32), v.astype(np.float16).astype(np.float32)
            self.k[il, n_past:T], self.v[il, n_past:T] = k.reshape(N, -1), v.reshape(N, -1)
            kc, vc = self.k[il, :T].reshape(T, HKV, D), self.v[il, :T].reshape(T, HKV, D)
            att = np.zeros((N, H, D), np.float32)
            for t in range(N):
                for h in range(H):
                    kk, vv = kc[:, h // G], vc[:, h // G]                                        # [T][D]
                    dot = np.zeros(T, np.float32)
                    for i in range(D):                                                           # dot += kk[i] * q[i], in order
                        dot = dot + kk[:, i] * q[t, h, i]
                    sc = dot * scale
                    sc[n_past + t + 1:] = -np.inf                                                # causal mask
                    sc = o.soft_max(sc)
                    acc = np.zeros(D, np.float32)
                    for pp in range(T):                                                          # acc += V[p] * sc[p], in order
                        acc = acc + vv[pp] * sc[pp]
                    att[t, h] = acc
            ao = self._mm(p + "self_attention.dense.weight", att.reshape(N, E))
            up = o.gelu(self._mm(p + "mlp.dense_h_to_4h.weight", xm))
            dn = self._mm(p + "mlp.dense_4h_to_h.weight", up)
            inp = (dn + ao) + inp
        rows = inp if all_logits else inp[-1:]
        xf = o.layernorm(rows, self._vec("transformer.ln_f.weight"), self._vec("transformer.ln_f.bias"))
        return self._mm("lm_head.weight", xf)
