"""ctypes wrapper of oracle/_ref/libfalcon_chain.so (ref_sample_chain.cpp, built by `make -C oracle -f sample_chain.mk` where the
reference sources exist): falcon_main's whole sampling chain through the reference's own llama_sample_* functions."""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libfalcon_chain.so")


def have_chain():
    return os.path.exists(LIB)


def have_stages():
    """the library exports refh_sample_chain_stages (a library built from an older ref_sample_chain.cpp does not)"""
    return have_chain() and hasattr(C.CDLL(LIB), "refh_sample_chain_stages")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class RefChain:
    """a reference context (its n_vocab is mirostat 1's N, its std::mt19937 drives the draws) plus the chain over caller rows"""

    def __init__(self, model_path, n_ctx=64):
        L = self.L = C.CDLL(LIB)
        L.refh_load.restype = C.c_void_p
        L.refh_load.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.refh_set_seed.argtypes = [C.c_void_p, C.c_int]
        L.refh_free.argtypes = [C.c_void_p]
        L.refh_n_vocab.argtypes = [C.c_void_p]
        L.refh_sample.restype = C.c_int
        L.refh_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
        L.refh_sample_chain.restype = C.c_int
        L.refh_sample_chain.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 7 + \
            [C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        self.h = L.refh_load(model_path.encode(), n_ctx, 8, 0, 0)
        if not self.h:
            raise RuntimeError("reference failed to load " + model_path)
        self.n_vocab = L.refh_n_vocab(self.h)

    def set_seed(self, seed):
        self.L.refh_set_seed(self.h, seed)

    def sample(self, logits, last_tokens, top_k, top_p, temp, repeat_penalty):
        """the existing default-chain harness (refh_sample), for comparison"""
        lg = np.ascontiguousarray(logits, np.float32)
        lt = np.ascontiguousarray(last_tokens, np.int32)
        return int(self.L.refh_sample(self.h, _p(lg), lg.size, _p(lt), lt.size, top_k, top_p, temp, repeat_penalty))

    def sample_chain(self, logits, last_tokens, mu, top_k=40, top_p=0.95, tfs_z=1.0, typical_p=1.0, temp=0.8, repeat_penalty=1.1,
                     frequency_penalty=0.0, presence_penalty=0.0, mirostat=0, mirostat_tau=5.0, mirostat_eta=0.1, logit_bias=None):
        """-> (id, mu after the step)"""
        lg = np.ascontiguousarray(logits, np.float32)
        lt = np.ascontiguousarray(last_tokens, np.int32)
        ids = np.array(list((logit_bias or {}).keys()), np.int32)
        vals = np.array(list((logit_bias or {}).values()), np.float32)
        m = C.c_float(mu)
        tok = self.L.refh_sample_chain(self.h, _p(lg), lg.size, _p(lt), lt.size, top_k, top_p, tfs_z, typical_p, temp, repeat_penalty,
                                       frequency_penalty, presence_penalty, mirostat, mirostat_tau, mirostat_eta, C.byref(m),
                                       ids.size, _p(ids), _p(vals))
        return int(tok), float(m.value)

    STAGES = ("row", "order", "tfs", "typical", "top_p", "temp", "final")

    def sample_chain_stages(self, logits, last_tokens, mu, top_k=40, top_p=0.95, tfs_z=1.0, typical_p=1.0, temp=0.8, repeat_penalty=1.1,
                            frequency_penalty=0.0, presence_penalty=0.0, mirostat=0, mirostat_tau=5.0, mirostat_eta=0.1, logit_bias=None):
        """-> (id, mu after the step, {stage: {"n", "ids", "logits", "p"}}): the candidates array after each llama_sample_* call of
        refh_sample_chain (ref_sample_chain.cpp); a stage no call reached is absent"""
        lg = np.ascontiguousarray(logits, np.float32)
        lt = np.ascontiguousarray(last_tokens, np.int32)
        ids = np.array(list((logit_bias or {}).keys()), np.int32)
        vals = np.array(list((logit_bias or {}).values()), np.float32)
        V = lg.size
        sizes = np.empty(7, np.int32)
        o_ids, o_l, o_p = np.empty(7 * V, np.int32), np.empty(7 * V, np.float32), np.empty(7 * V, np.float32)
        f = self.L.refh_sample_chain_stages
        f.restype, f.argtypes = C.c_int, self.L.refh_sample_chain.argtypes + [C.c_void_p] * 4
        m = C.c_float(mu)
        tok = f(self.h, _p(lg), V, _p(lt), lt.size, top_k, top_p, tfs_z, typical_p, temp, repeat_penalty,
                                              frequency_penalty, presence_penalty, mirostat, mirostat_tau, mirostat_eta, C.byref(m),
                                              ids.size, _p(ids), _p(vals), _p(sizes), _p(o_ids), _p(o_l), _p(o_p))
        st = {}
        for s, name in enumerate(self.STAGES):
            n = int(sizes[s])
            if n >= 0:
                st[name] = dict(n=n, ids=o_ids[s * V:s * V + n].copy(), logits=o_l[s * V:s * V + n].copy(), p=o_p[s * V:s * V + n].copy())
        return int(tok), float(m.value), st

    def close(self):
        if self.h:
            self.L.refh_free(self.h)
            self.h = None
