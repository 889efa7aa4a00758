"""ctypes binding of csrc/libggml_b200.so (the C ABI declared in include/ggml_b200.h).

Used by tests/ and bench.py only; the library itself has no Python dependency.  There is no fallback of any
kind: if the CUDA library is missing or no sm_90 GPU is visible, loading / init fails loudly.
"""
import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libggml_b200.so")

# every symbol include/ggml_b200.h declares (checked by tests/test_abi.py against the header text)
PART_A = ["b200_event_create", "b200_event_destroy", "b200_event_record", "b200_event_synchronize", "b200_event_elapsed_ms",
          "b200_stream_synchronize", "b200_init", "b200_device_count", "b200_set_stream", "b200_synchronize", "b200_malloc", "b200_free", "b200_memcpy_h2d",
          "b200_memcpy_d2h", "b200_memset", "b200_host_malloc", "b200_host_free", "b200_weight_upload", "b200_weight_random",
          "b200_weight_free", "b200_weight_device_bytes", "b200_dequantize_rows", "b200_actq_alloc", "b200_actq_free",
          "b200_quantize_act", "b200_actq_download", "b200_actq_alloc_f16", "b200_actq_download_f16", "b200_actq_to_f16", "b200_mul_mat", "b200_mul_mat_f16", "b200_mul_mat_vec_q", "b200_mul_mat_vec_q_chain", "b200_quantize_weights", "b200_quantize_weights_rows", "b200_quantize_chunks", "b200_mmv_max_n", "b200_mmv_launch_shape", "b200_gemm_launch_shape", "b200_layernorm",
          "b200_gelu", "b200_add", "b200_rope_neox", "b200_attention", "b200_layernorm_q", "b200_attention_decode", "b200_attention_kv16", "b200_attention_decode_kv16",
          "b200_sampler_create", "b200_sampler_create_chain", "b200_sampler_sample", "b200_sampler_mirostat_mu", "b200_sampler_free",
          "b200_sampler_tap", "b200_sampler_tap_read", "b200_token_nll"]
PART_B = ["b200_falcon_create", "b200_falcon_create_kv", "b200_falcon_create_streamed", "b200_falcon_stream_info", "b200_falcon_kv_type", "b200_falcon_kv_device_bytes", "b200_falcon_set_tensor", "b200_falcon_set_tensor_random", "b200_falcon_load_ggcc",
          "b200_ggcc_read_hparams", "b200_quantize_ggcc", "b200_falcon_free", "b200_falcon_weight_bytes", "b200_nccl_unique_id",
          "b200_falcon_init_pipeline", "b200_falcon_eval", "b200_falcon_decode_dev", "b200_falcon_logits_dev", "b200_falcon_generate_greedy",
          "b200_falcon_last_launches", "b200_attention_long_launches", "b200_falcon_last_ms", "b200_falcon_stream", "b200_falcon_profile_matvec",
          "b200_falcon_kv_read", "b200_falcon_kv_write", "b200_falcon_kv_shadow_read", "b200_falcon_kv_fill_random", "b200_falcon_generate", "b200_falcon_generate_chain", "b200_falcon_load_seconds", "b200_falcon_save_kv", "b200_falcon_load_kv",
          "b200_falcon_tap", "b200_falcon_tap_layers", "b200_falcon_tap_read", "b200_falcon_score", "b200_falcon_perplexity", "b200_falcon_set_embeddings", "b200_falcon_embeddings"]


def build(verbose=False):
    """nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo for every .cu (csrc/Makefile); cross-compiles without a GPU."""
    subprocess.check_call(["make", "-C", CSRC, "-j8"] + ([] if verbose else ["-s"]))
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libggml_b200.so is not built (run __graft_entry__.build()); there is no CPU fallback")
        L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        vp, i32, i64, f32, sz = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t
        sig = {
            "b200_init": (i32, [i32]), "b200_device_count": (i32, []), "b200_set_stream": (None, [vp]), "b200_synchronize": (None, []),
            "b200_event_create": (vp, []), "b200_event_destroy": (None, [vp]), "b200_event_record": (None, [vp, vp]),
            "b200_event_synchronize": (None, [vp]), "b200_event_elapsed_ms": (f32, [vp, vp]), "b200_stream_synchronize": (None, [vp]),
            "b200_malloc": (vp, [sz]), "b200_free": (None, [vp]), "b200_memcpy_h2d": (None, [vp, vp, sz]), "b200_memcpy_d2h": (None, [vp, vp, sz]),
            "b200_memset": (None, [vp, i32, sz]), "b200_host_malloc": (vp, [sz]), "b200_host_free": (None, [vp]),
            "b200_weight_upload": (vp, [i32, i64, i64, vp]), "b200_weight_random": (vp, [i32, i64, i64, C.c_uint64]),
            "b200_weight_free": (None, [vp]), "b200_weight_device_bytes": (sz, [vp]),
            "b200_dequantize_rows": (None, [vp, vp, i32, vp, i64]),
            "b200_actq_alloc": (vp, [i32, i64, i32]), "b200_actq_free": (None, [vp]), "b200_quantize_act": (None, [vp, i64, vp]),
            "b200_actq_download": (None, [vp, vp, vp, vp, vp]),
            "b200_actq_alloc_f16": (vp, [i32, i64, i32]), "b200_actq_download_f16": (None, [vp, vp]), "b200_actq_to_f16": (None, [vp, vp, i64]),
            "b200_mul_mat": (None, [vp, vp, i64, i32, vp, i64]), "b200_mul_mat_vec_q": (None, [vp, vp, vp, i64, i32, vp, vp]),
            "b200_mmv_max_n": (i32, []), "b200_mmv_launch_shape": (i32, [i32, i64, vp]), "b200_gemm_launch_shape": (i32, [i32, i64, i64, i32, i64, i32, vp]),"b200_mul_mat_vec_q_chain": (i32, [vp, vp, vp, i32, vp]), "b200_quantize_weights": (i32, [i32, vp, vp, i64]), "b200_quantize_weights_rows": (i32, [i32, vp, vp, i64, i64]),
            "b200_quantize_chunks": (i64, [i32, vp, vp, i64, i64, vp]), "b200_quantize_ggcc": (i32, [C.c_char_p, C.c_char_p, vp, vp]), "b200_mul_mat_f16": (i32, [vp, vp, i64, i32, vp, i64, i32, i32]),
            "b200_layernorm": (None, [vp, i64, vp, vp, vp, i64, i32, i32]), "b200_gelu": (None, [vp, vp, i64]), "b200_add": (None, [vp, vp, vp, i64]),
            "b200_rope_neox": (None, [vp, i32, i32, i32, i64, i32, i32, i32, f32, i32]),
            "b200_attention": (None, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32]),
            "b200_layernorm_q": (None, [vp, i64, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32]),
            "b200_attention_decode": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
            "b200_attention_kv16": (None, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32]),
            "b200_attention_decode_kv16": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
            "b200_falcon_kv_read": (i32, [vp, i32, i32, i32, vp, vp]), "b200_falcon_kv_write": (i32, [vp, i32, i32, i32, vp, vp]),
            "b200_falcon_kv_shadow_read": (i32, [vp, i32, i32, i32, vp, vp]),
            "b200_falcon_kv_fill_random": (i32, [vp, i32, i32, C.c_uint64]),
            "b200_sampler_create": (vp, [vp, vp, i32]), "b200_sampler_sample": (i32, [vp, vp, i32]), "b200_sampler_free": (None, [vp]),
            "b200_sampler_create_chain": (vp, [vp, vp, i32]), "b200_sampler_mirostat_mu": (f32, [vp]),
            "b200_sampler_tap": (i32, [vp, i32]), "b200_sampler_tap_read": (i32, [vp, C.c_char_p, C.c_char_p, vp, sz]),
            "b200_falcon_generate": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
            "b200_falcon_generate_chain": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
            "b200_falcon_load_seconds": (C.c_double, [vp, vp]),
            "b200_falcon_save_kv": (i32, [vp, C.c_char_p, i32]), "b200_falcon_load_kv": (i32, [vp, C.c_char_p]),
            "b200_falcon_create": (vp, [vp]), "b200_falcon_create_kv": (vp, [vp, i32]), "b200_falcon_kv_type": (i32, [vp]),
            "b200_falcon_create_streamed": (vp, [vp, i32, vp, i32]), "b200_falcon_stream_info": (i32, [vp, vp, vp, vp, vp]),
            "b200_falcon_kv_device_bytes": (sz, [vp]), "b200_falcon_set_tensor": (None, [vp, C.c_char_p, i32, i32, vp, vp]),
            "b200_falcon_set_tensor_random": (None, [vp, C.c_char_p, i32, C.c_uint64]),
            "b200_falcon_load_ggcc": (i32, [vp, C.c_char_p]), "b200_ggcc_read_hparams": (i32, [C.c_char_p, vp]),
            "b200_falcon_free": (None, [vp]), "b200_falcon_weight_bytes": (sz, [vp]),
            "b200_nccl_unique_id": (None, [vp]), "b200_falcon_init_pipeline": (None, [vp, vp]),
            "b200_falcon_eval": (i32, [vp, vp, i32, i32, i32, vp, i32]), "b200_falcon_decode_dev": (i32, [vp, vp, i32, i32]), "b200_falcon_generate_greedy": (i32, [vp, i32, i32, i32, i32, vp]),
            "b200_falcon_logits_dev": (vp, [vp]), "b200_falcon_last_launches": (i32, [vp]), "b200_falcon_last_ms": (f32, [vp]),
            "b200_falcon_stream": (vp, [vp]), "b200_falcon_profile_matvec": (f32, [vp, i32, vp, vp]),
            "b200_falcon_tap": (i32, [vp, i32]), "b200_falcon_tap_layers": (i32, [vp, vp, i32]), "b200_falcon_tap_read": (i32, [vp, i32, C.c_char_p, vp, sz]),
            "b200_token_nll": (None, [vp, i32, i32, i64, vp, vp, vp]),
            "b200_falcon_score": (i32, [vp, vp, i32, i32, i32, vp, vp]), "b200_falcon_perplexity": (i32, [vp, vp, i32, i32, vp, vp]),
            "b200_falcon_set_embeddings": (i32, [vp, i32]), "b200_falcon_embeddings": (C.POINTER(C.c_float), [vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        L.b200_surface_takeover_evals.restype, L.b200_surface_takeover_evals.argtypes = C.c_long, []      # ggml_surface.cu test hook
        L.b200_attention_long_launches.restype, L.b200_attention_long_launches.argtypes = C.c_int, []
        _lib = L
    return _lib


_inited = False


def init(device=None):
    global _inited
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    L = lib()
    if L.b200_device_count() <= 0:
        raise RuntimeError("no CUDA device visible: libggml_b200 has no CPU fallback")
    sms = L.b200_init(device)
    _inited = True
    return sms


def _np_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def mmv_launch_shape(wtype, K):
    """-> (threads per CTA, pieces per thread, ring depth) of the tuned decode mat-vec, or None for the generic kernel."""
    s = (C.c_int * 3)()
    return tuple(s) if lib().b200_mmv_launch_shape(wtype, K, s) else None


def gemm_launch_shape(wtype, K, M, N, x_stride=None, gelu=False):
    """-> (BN, ksplit, producer) of the wgmma prompt GEMM for one call of at most 512 tokens (producer: the weight type of a dedicated
    dequantiser, or -1 for the generic one), or None when the CUDA-core kernel runs"""
    s = (C.c_int * 3)()
    return tuple(s) if lib().b200_gemm_launch_shape(wtype, K, M, N, x_stride or K, int(bool(gelu)), s) else None


class DevBuf:
    """A device allocation with numpy-typed upload/download helpers."""

    def __init__(self, nbytes=None, src=None):
        self.L = lib()
        if src is not None:
            src = np.ascontiguousarray(src)
            nbytes = src.nbytes
        self.nbytes = int(nbytes)
        self.ptr = self.L.b200_malloc(self.nbytes)
        if src is not None:
            self.L.b200_memcpy_h2d(self.ptr, _np_ptr(src), self.nbytes)

    def upload(self, a):
        a = np.ascontiguousarray(a)
        assert a.nbytes <= self.nbytes
        self.L.b200_memcpy_h2d(self.ptr, _np_ptr(a), a.nbytes)

    def download(self, dtype, shape):
        out = np.empty(shape, dtype=dtype)
        assert out.nbytes <= self.nbytes
        self.L.b200_memcpy_d2h(_np_ptr(out), self.ptr, out.nbytes)
        return out

    def zero(self):
        self.L.b200_memset(self.ptr, 0, self.nbytes)

    def free(self):
        if self.ptr:
            self.L.b200_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def token_nll(logits_dev, n_vocab, n_rows, targets_dev, nll_dev, row_stride=None, stream=None):
    """b200_token_nll: -log(softmax(row r)[targets[r]]) of device rows logits_dev + r * row_stride into nll_dev[r] (device pointers;
    target -1 leaves nll_dev[r] as it is, any other target outside [0, n_vocab) writes NaN), enqueued on `stream` (None: the backend's)"""
    lib().b200_token_nll(logits_dev, n_vocab, n_rows, row_stride or n_vocab, targets_dev, nll_dev, stream)


class Weight:
    def __init__(self, ggml_type, K, M, blocks=None, seed=None):
        self.L = lib()
        self.type, self.K, self.M = ggml_type, K, M
        if blocks is not None:
            blocks = np.ascontiguousarray(blocks)
            self.h = self.L.b200_weight_upload(ggml_type, K, M, _np_ptr(blocks))
        else:
            self.h = self.L.b200_weight_random(ggml_type, K, M, seed or 1)

    def dequantize(self, rows=None):
        if rows is None:
            n, rp = self.M, None
        else:
            rows = np.ascontiguousarray(rows, dtype=np.int32)
            rb = DevBuf(src=rows)
            n, rp = rows.size, rb.ptr
        out = DevBuf(n * self.K * 4)
        self.L.b200_dequantize_rows(self.h, rp, n, out.ptr, self.K)
        return out.download(np.float32, (n, self.K))

    def free(self):
        if self.h:
            self.L.b200_weight_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class ActQ:
    """quantised activation rows; f16=True adds the fp16 GEMM-operand plane fp16(d * q) that every producer then fills too"""

    def __init__(self, wtype, K, N, f16=False):
        self.L = lib()
        self.wtype, self.K, self.N = wtype, K, N
        self.h = (self.L.b200_actq_alloc_f16 if f16 else self.L.b200_actq_alloc)(wtype, K, N)

    def quantize(self, x_dev, x_stride=None):
        self.L.b200_quantize_act(x_dev, x_stride or self.K, self.h)

    def download(self):
        kq = self.wtype >= 10
        blk = 256 if kq else 32
        q = np.empty((self.N, self.K), np.int8)
        d = np.empty((self.N, self.K // blk), np.float32)
        s = np.empty((self.N, self.K // 32), np.float32)
        bs = np.empty((self.N, self.K // (16 if kq else 32)), np.int16)
        self.L.b200_actq_download(self.h, _np_ptr(q), _np_ptr(d), _np_ptr(s), _np_ptr(bs))
        return q, d, s, bs

    def download_f16(self):
        """-> the fp16 plane [N][K] (the ActQ must have been made with f16=True)"""
        h = np.empty((self.N, self.K), np.float16)
        self.L.b200_actq_download_f16(self.h, _np_ptr(h))
        return h

    def to_f16(self, buf, stride=None):
        """fp16(d * q) of the codes and scales into the DevBuf `buf` [N][stride] (actq_to_f16: the GEMM operand built separately)"""
        self.L.b200_actq_to_f16(self.h, buf.ptr, stride or self.K)

    def free(self):
        if self.h:
            self.L.b200_actq_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class SamplingParams(C.Structure):
    """b200_sampling_params: falcon_main's defaults (examples/falcon_common.h: top_k 40, top_p 0.95, temp 0.8, repeat_penalty 1.1, repeat_last_n 64)"""
    _fields_ = [("top_k", C.c_int32), ("top_p", C.c_float), ("temp", C.c_float), ("repeat_penalty", C.c_float), ("repeat_last_n", C.c_int32), ("seed", C.c_uint32)]

    def __init__(self, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, repeat_last_n=64, seed=1):
        super().__init__(top_k, top_p, temp, repeat_penalty, repeat_last_n, seed)


class SamplingChain(C.Structure):
    """b200_sampling_chain: falcon_main's whole chain with its defaults (examples/falcon_common.h:40-52); top_k <= 0 is the whole
    vocabulary, logit_bias a {id: value} mapping (value may be -inf: falcon_main's --ignore-eos)"""
    _fields_ = [("top_k", C.c_int32), ("top_p", C.c_float), ("tfs_z", C.c_float), ("typical_p", C.c_float), ("temp", C.c_float),
                ("repeat_penalty", C.c_float), ("frequency_penalty", C.c_float), ("presence_penalty", C.c_float),
                ("repeat_last_n", C.c_int32), ("mirostat", C.c_int32), ("mirostat_tau", C.c_float), ("mirostat_eta", C.c_float),
                ("seed", C.c_uint32), ("n_logit_bias", C.c_int32), ("logit_bias_ids", C.c_void_p), ("logit_bias_values", C.c_void_p)]

    def __init__(self, top_k=40, top_p=0.95, tfs_z=1.0, typical_p=1.0, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0,
                 presence_penalty=0.0, repeat_last_n=64, mirostat=0, mirostat_tau=5.0, mirostat_eta=0.1, seed=1, logit_bias=None):
        ids = np.array(list((logit_bias or {}).keys()), np.int32)
        vals = np.array(list((logit_bias or {}).values()), np.float32)
        self._bias = (ids, vals)                                    # kept alive with the struct
        super().__init__(top_k, top_p, tfs_z, typical_p, temp, repeat_penalty, frequency_penalty, presence_penalty, repeat_last_n,
                         mirostat, mirostat_tau, mirostat_eta, seed, ids.size, ids.ctypes.data if ids.size else None,
                         vals.ctypes.data if vals.size else None)


class Sampler:
    """stand-alone device sampler over logits rows in HBM (b200_sampler_*); params: SamplingParams or SamplingChain"""

    def __init__(self, params, last_tokens=()):
        self.L = lib()
        lt = np.ascontiguousarray(last_tokens, dtype=np.int32)
        create = self.L.b200_sampler_create_chain if isinstance(params, SamplingChain) else self.L.b200_sampler_create
        self.h = create(C.byref(params), _np_ptr(lt) if lt.size else None, lt.size)
        if not self.h:
            raise ValueError("b200_sampler_create: bad sampling parameters")

    def sample(self, logits_dev_ptr, n_vocab):
        return int(self.L.b200_sampler_sample(self.h, logits_dev_ptr, n_vocab))

    def mirostat_mu(self):
        return float(self.L.b200_sampler_mirostat_mu(self.h))

    def tap(self, on=True):
        """switch the stage tap on (copies of the candidate list after every stage, b200_sampler_tap) or off"""
        if self.L.b200_sampler_tap(self.h, int(bool(on))) != 0:
            raise RuntimeError("b200_sampler_tap failed")

    def _tap_field(self, stage, field, dtype, count):
        out = np.empty(count, dtype)
        if self.L.b200_sampler_tap_read(self.h, stage.encode(), field.encode(), _np_ptr(out), out.nbytes) != 0:
            raise KeyError("b200_sampler_tap_read: no field %r of stage %r with %d bytes" % (field, stage, out.nbytes))
        return out

    def tap_stages(self, n_vocab):
        """every stage of the most recent sample: {stage: {field: value}}; a stage that did not run has n = -1 only"""
        st = {"row": {"n": n_vocab, "logits": self._tap_field("row", "logits", np.float32, n_vocab)}}
        for stage in ("order", "tfs", "typical", "top_p", "temp", "final"):
            n = int(self._tap_field(stage, "n", np.int32, 1)[0])
            d = st[stage] = {"n": n}
            if n < 0:
                continue
            d["ids"] = self._tap_field(stage, "ids", np.int32, n)
            d["logits"] = self._tap_field(stage, "logits", np.float32, n)
            if stage not in ("order", "temp"):
                d["p"] = self._tap_field(stage, "p", np.float32, n)
        st["typical"]["entropy"] = np.float32(self._tap_field("typical", "entropy", np.float32, 1)[0])
        f = st["final"]
        f["u"] = float(self._tap_field("final", "u", np.float64, 1)[0])
        for k in ("pick", "id", "k"):
            f[k] = int(self._tap_field("final", k, np.int32, 1)[0])
        f["mu"] = np.float32(self._tap_field("final", "mu", np.float32, 1)[0])
        return st

    def free(self):
        if self.h:
            self.L.b200_sampler_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def quantize_chunks(ggml_type, x_dev, dst_dev, n_elems, chunk_elems, hist=None):
    """b200_quantize_chunks: ggml_quantize_chunk over consecutive chunks of chunk_elems values (device pointers).  hist: an int64[16]
    array the legacy code histograms are added to, or None.  -> bytes written, 0 for an unsupported type, -1 for a bad shape"""
    hp = None
    if hist is not None:
        assert hist.dtype == np.int64 and hist.size == 16 and hist.flags.c_contiguous
        hp = _np_ptr(hist)
    return int(lib().b200_quantize_chunks(ggml_type, x_dev, dst_dev, n_elems, chunk_elems, hp))


class QuantizeParams(C.Structure):
    """b200_quantize_params: llama_model_quantize_params (nthread <= 0: the host's hardware threads)"""
    _fields_ = [("nthread", C.c_int32), ("ftype", C.c_int32), ("allow_requantize", C.c_int32), ("quantize_output_tensor", C.c_int32)]


class QuantizeReport(C.Structure):
    _fields_ = [("size_org", C.c_uint64), ("size_new", C.c_uint64), ("hist", C.c_int64 * 16), ("n_tensors", C.c_int32),
                ("n_quantized", C.c_int32), ("seconds", C.c_double), ("staging_bytes", C.c_uint64), ("device_bytes", C.c_uint64)]


def quantize_ggcc(path_in, path_out, ftype, nthread=0, allow_requantize=False, quantize_output_tensor=True):
    """b200_quantize_ggcc: falcon_quantize on the device -> (return code, QuantizeReport).  0: written; 1: the reference refuses
    (unknown ftype, a k-quant of a row length not a multiple of 256, requantisation without allow_requantize); -1: unreadable or
    malformed input, or an I/O error"""
    p = QuantizeParams(nthread, ftype, int(bool(allow_requantize)), int(bool(quantize_output_tensor)))
    r = QuantizeReport()
    rc = lib().b200_quantize_ggcc(path_in.encode(), path_out.encode(), C.byref(p), C.byref(r))
    return int(rc), r


class FalconParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "falcon_type", "n_ctx", "n_batch",
                                          "layer_first", "layer_last", "rank", "world")]


def layer_range(n_layer, rank, world):
    """contiguous layer ranges, remainder spread over the first ranks"""
    base, rem = divmod(n_layer, world)
    first = rank * base + min(rank, rem)
    return first, first + base + (1 if rank < rem else 0)


class Falcon:
    """The Falcon eval path (include/ggml_b200.h part B)."""

    def __init__(self, hp, n_ctx, n_batch=1, rank=0, world=1, layers=None, kv_f16=False, streamed=()):
        """kv_f16: keep the KV cache in fp16 (b200_falcon_create_kv with GGML_TYPE_F16, the reference's f16_kv): half the cache bytes,
        K / V rounded to fp16 as they are stored.  streamed: global indices of layers whose matrices stay in pinned host memory and are
        copied to the device for every eval (b200_falcon_create_streamed), for models larger than the card's memory"""
        self.L = lib()
        self.hp = dict(hp)
        lf, ll = layers if layers is not None else layer_range(hp["n_layer"], rank, world)      # layers: an explicit (first, last) range, e.g. balanced by bytes
        self.params = FalconParams(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["falcon_type"],
                                   n_ctx, n_batch, lf, ll, rank, world)
        self.layer_first, self.layer_last, self.rank, self.world = lf, ll, rank, world
        streamed = np.ascontiguousarray(streamed, dtype=np.int32)
        if streamed.size:
            self.h = self.L.b200_falcon_create_streamed(C.byref(self.params), 1 if kv_f16 else 0, _np_ptr(streamed), streamed.size)
            if not self.h:
                raise ValueError("b200_falcon_create_streamed: streamed layers %s outside [%d, %d) or repeated, or world > 1"
                                 % (streamed.tolist(), lf, ll))
        else:
            self.h = self.L.b200_falcon_create_kv(C.byref(self.params), 1 if kv_f16 else 0)
        self.n_vocab = hp["n_vocab"]

    @staticmethod
    def read_hparams(path):
        p = FalconParams()
        if lib().b200_ggcc_read_hparams(path.encode(), C.byref(p)) != 0:
            raise ValueError("not a GGCC v10 file: " + path)
        return {k: getattr(p, k) for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "falcon_type")}

    def load_ggcc(self, path):
        if self.L.b200_falcon_load_ggcc(self.h, path.encode()) != 0:
            raise RuntimeError("failed to load " + path)

    def load_stats(self):
        """-> (seconds, quantised-matrix bytes) of the last load_ggcc"""
        by = C.c_size_t(0)
        return float(self.L.b200_falcon_load_seconds(self.h, C.byref(by))), by.value

    def set_tensor(self, name, ggml_type, ne, data):
        data = np.ascontiguousarray(data)
        ne_a = (C.c_int64 * 2)(ne[0], ne[1] if len(ne) > 1 else 1)
        self.L.b200_falcon_set_tensor(self.h, name.encode(), ggml_type, len(ne), ne_a, _np_ptr(data))

    def set_tensors(self, tensors):
        for name, (t, ne, arr) in tensors.items():
            self.set_tensor(name, t, ne, arr)

    def set_random(self, shapes, wtype, seed=1):
        """random-init every tensor of `shapes` ({name: ne}) on the device: 2-D as `wtype` blocks, 1-D as f32"""
        for i, (name, ne) in enumerate(shapes.items()):
            self.L.b200_falcon_set_tensor_random(self.h, name.encode(), wtype if len(ne) == 2 else 0, seed * 1000003 + i)

    def eval(self, tokens, n_past, n_ctx_rope=0, all_logits=False):
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        out = np.zeros((tokens.size if all_logits else 1, self.n_vocab), dtype=np.float32)
        rc = self.L.b200_falcon_eval(self.h, _np_ptr(tokens), tokens.size, n_past, n_ctx_rope, _np_ptr(out), int(all_logits))
        if rc != 0:
            raise RuntimeError("b200_falcon_eval failed (rc=%d)" % rc)
        return out

    def set_embeddings(self, on=True):
        """falcon_context_params.embedding: every eval also returns the last token's final LayerNorm row (b200_falcon_set_embeddings)"""
        if self.L.b200_falcon_set_embeddings(self.h, int(bool(on))) != 0:
            raise RuntimeError("b200_falcon_set_embeddings: this rank has no head")

    def embeddings(self):
        """-> a copy of the n_embd floats of the most recent eval's "result_norm" row (falcon_get_embeddings), or None when embeddings
        are off or the most recent eval call was not b200_falcon_eval"""
        p = self.L.b200_falcon_embeddings(self.h)
        return np.ctypeslib.as_array(p, (self.hp["n_embd"],)).copy() if p else None

    def score(self, tokens, n_past, targets, n_ctx_rope=0):
        """b200_falcon_score: evaluate `tokens` at n_past and return the terms -log p(targets[i]) as float32 [n_tokens], NaN where
        targets[i] == -1 (not scored); no logits leave the device"""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        targets = np.ascontiguousarray(targets, dtype=np.int32)
        if targets.size != tokens.size:
            raise ValueError("score: %d targets for %d tokens" % (targets.size, tokens.size))
        out = np.full(tokens.size, np.nan, np.float32)
        rc = self.L.b200_falcon_score(self.h, _np_ptr(tokens), tokens.size, n_past, n_ctx_rope, _np_ptr(targets), _np_ptr(out))
        if rc != 0:
            raise RuntimeError("b200_falcon_score failed (rc=%d)" % rc)
        return out

    def perplexity(self, tokens, n_ctx):
        """b200_falcon_perplexity: falcon_perplexity over `tokens` in chunks of n_ctx -> (ppl after each chunk as float64 [n_chunk],
        the per-token terms as float32 [n_chunk * (n_ctx - 1 - min(512, n_ctx // 2))])"""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        n_chunk = tokens.size // n_ctx if n_ctx > 0 else 0
        ppl = np.zeros(max(n_chunk, 1), np.float64)
        nll = np.zeros(max(n_chunk * max(n_ctx - 1 - min(512, n_ctx // 2), 0), 1), np.float32)
        rc = self.L.b200_falcon_perplexity(self.h, _np_ptr(tokens), tokens.size, n_ctx, _np_ptr(ppl), _np_ptr(nll))
        if rc < 0:
            raise RuntimeError("b200_falcon_perplexity: bad n_ctx / tokens, or a pipeline engine")
        return ppl[:rc], nll[:rc * max(n_ctx - 1 - min(512, n_ctx // 2), 0)]

    def generate_greedy(self, first_token, n_past, n_steps, n_ctx_rope=0):
        out = np.zeros(n_steps, dtype=np.int32)
        rc = self.L.b200_falcon_generate_greedy(self.h, int(first_token), n_past, n_steps, n_ctx_rope, _np_ptr(out))
        if rc != 0:
            raise RuntimeError("b200_falcon_generate_greedy failed (rc=%d)" % rc)
        return out

    def generate(self, params, last_tokens, first_token, n_past, n_steps, n_ctx_rope=0):
        """generation with the sampling chain on the device (b200_falcon_generate); last_tokens seed the repetition-penalty window"""
        out = np.zeros(n_steps, dtype=np.int32)
        lt = np.ascontiguousarray(last_tokens, dtype=np.int32)
        rc = self.L.b200_falcon_generate(self.h, C.byref(params), _np_ptr(lt) if lt.size else None, lt.size, int(first_token), n_past, n_steps, n_ctx_rope, _np_ptr(out))
        if rc != 0:
            raise RuntimeError("b200_falcon_generate failed (rc=%d)" % rc)
        return out

    def generate_chain(self, chain, last_tokens, first_token, n_past, n_steps, n_ctx_rope=0):
        """generation with the whole sampling chain on the device (b200_falcon_generate_chain; chain: SamplingChain)"""
        out = np.zeros(n_steps, dtype=np.int32)
        lt = np.ascontiguousarray(last_tokens, dtype=np.int32)
        rc = self.L.b200_falcon_generate_chain(self.h, C.byref(chain), _np_ptr(lt) if lt.size else None, lt.size, int(first_token), n_past, n_steps, n_ctx_rope, _np_ptr(out))
        if rc != 0:
            raise RuntimeError("b200_falcon_generate_chain failed (rc=%d)" % rc)
        return out

    def decode_dev(self, token_dev_ptr, n_past, n_ctx_rope=0):
        if self.L.b200_falcon_decode_dev(self.h, token_dev_ptr, n_past, n_ctx_rope) != 0:
            raise RuntimeError("b200_falcon_decode_dev: n_past %d outside [0, n_ctx)" % n_past)

    def kv_read(self, layer, pos, n):
        """-> (K, V) rows [pos, pos + n) of `layer`, each float32 [n][n_head_kv * head_dim]"""
        w = self.hp["n_head_kv"] * (self.hp["n_embd"] // self.hp["n_head"])
        k, v = np.empty((n, w), np.float32), np.empty((n, w), np.float32)
        if self.L.b200_falcon_kv_read(self.h, layer, pos, n, _np_ptr(k), _np_ptr(v)) != 0:
            raise RuntimeError("b200_falcon_kv_read: bad layer / range")
        return k, v

    def kv_write(self, layer, pos, k, v):
        k, v = np.ascontiguousarray(k, np.float32), np.ascontiguousarray(v, np.float32)
        if self.L.b200_falcon_kv_write(self.h, layer, pos, k.shape[0], _np_ptr(k), _np_ptr(v)) != 0:
            raise RuntimeError("b200_falcon_kv_write: bad layer / range")

    def kv_shadow_read(self, layer, pos, n):
        """-> (k16 [n][n_head_kv][head_dim], vt16 [n_head_kv][head_dim][n]) of the fp16 cache copy, as uint16 bit patterns"""
        hkv, hd = self.hp["n_head_kv"], self.hp["n_embd"] // self.hp["n_head"]
        k, vt = np.empty((n, hkv, hd), np.uint16), np.empty((hkv, hd, n), np.uint16)
        if self.L.b200_falcon_kv_shadow_read(self.h, layer, pos, n, _np_ptr(k), _np_ptr(vt)) != 0:
            raise RuntimeError("b200_falcon_kv_shadow_read: no fp16 copy, bad layer or range")
        return k, vt

    def tap(self, on=True):
        """switch the test tap on (copies of every layer's intermediates, b200_falcon_tap) or off"""
        if self.L.b200_falcon_tap(self.h, int(bool(on))) != 0:
            raise RuntimeError("b200_falcon_tap failed")

    def tap_layers(self, layers):
        """switch the test tap on for the listed (global index) layers only (b200_falcon_tap_layers); the head is tapped too"""
        ids = np.ascontiguousarray(layers, dtype=np.int32)
        if self.L.b200_falcon_tap_layers(self.h, _np_ptr(ids), ids.size) != 0:
            raise RuntimeError("b200_falcon_tap_layers: a layer that is not local or listed twice")

    def tap_read(self, layer, node, dtype, shape):
        """-> one tapped buffer of the most recent eval (layer -1: after the head) as an array of `dtype` and `shape`"""
        out = np.empty(shape, dtype)
        if self.L.b200_falcon_tap_read(self.h, layer, node.encode(), _np_ptr(out), out.nbytes) != 0:
            raise KeyError("b200_falcon_tap_read: no node %r of layer %d with %d bytes" % (node, layer, out.nbytes))
        return out

    def save_kv(self, path, n_tokens):
        if self.L.b200_falcon_save_kv(self.h, path.encode(), n_tokens) != 0:
            raise RuntimeError("b200_falcon_save_kv failed")

    def load_kv(self, path):
        n = self.L.b200_falcon_load_kv(self.h, path.encode())
        if n < 0:
            raise RuntimeError("b200_falcon_load_kv: missing / truncated / mismatching session file")
        return n

    def kv_type(self):
        """-> 0 (f32 cache) or 1 (fp16 cache)"""
        return self.L.b200_falcon_kv_type(self.h)

    def kv_device_bytes(self):
        """-> device bytes of the KV cache plus its fp16 copies, all local layers"""
        return self.L.b200_falcon_kv_device_bytes(self.h)

    def kv_fill_random(self, pos, n, seed=1):
        if self.L.b200_falcon_kv_fill_random(self.h, pos, n, seed) != 0:
            raise RuntimeError("b200_falcon_kv_fill_random: bad range")

    def logits_dev(self):
        return self.L.b200_falcon_logits_dev(self.h)

    def stream(self):
        return self.L.b200_falcon_stream(self.h)

    def stream_info(self):
        """-> dict(layers, host_bytes, slot_bytes, copy_bytes) of the streamed layers (b200_falcon_stream_info)"""
        n = self.L.b200_falcon_stream_info(self.h, None, None, None, None)
        ids = np.zeros(max(n, 1), np.int32)
        hb, sb, cb = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        self.L.b200_falcon_stream_info(self.h, _np_ptr(ids), C.byref(hb), C.byref(sb), C.byref(cb))
        return dict(layers=ids[:n].tolist(), host_bytes=hb.value, slot_bytes=sb.value, copy_bytes=cb.value)

    def weight_bytes(self):
        return self.L.b200_falcon_weight_bytes(self.h)

    def last_launches(self):
        return self.L.b200_falcon_last_launches(self.h)

    def last_ms(self):
        return self.L.b200_falcon_last_ms(self.h)

    def profile_matvec(self, reps=3):
        """-> (total ms, launches, algorithmic bytes) of every resident mat-vec launched back to back"""
        n, by = C.c_int(0), C.c_size_t(0)
        ms = self.L.b200_falcon_profile_matvec(self.h, reps, C.byref(n), C.byref(by))
        return ms, n.value, by.value

    def init_pipeline(self, id_bytes):
        buf = (C.c_char * 128).from_buffer_copy(id_bytes)
        self.L.b200_falcon_init_pipeline(self.h, buf)

    @staticmethod
    def nccl_unique_id():
        buf = (C.c_char * 128)()
        lib().b200_nccl_unique_id(buf)
        return bytes(buf)

    def free(self):
        if self.h:
            self.L.b200_falcon_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
