"""-m gpu: every eval path of the Falcon engine, node by node, through the checker of tests/engine_nodes.py.

Each case runs its evals twice from the same KV state: once with the test tap off, once with it on (b200_falcon_tap).
  (h) logits and the KV cache must be bit-identical between the two runs: the tap's copies change nothing but timing;
  (a)-(g) must hold for every layer of every eval of the tapped run.
Tiny models (n_layer 2) cover the tuned mat-vec types (Q4_K, Q4_0, Q3_K), the generic mat-vec (Q6_K, Q5_1) and the generic paths
(F16 weights, mixed types, an F16 lm_head), each as an 8-token prompt (mat-vec batch), a 40-token prompt with n_batch 64 (GEMM, wgmma
prompt attention, fp16 shadow), decode steps by graph and eagerly, decode without the fused path, and decode across the long-context
attention tier.  The 2-layer, vocabulary-2048 models at real widths (test_real_geometry_gpu.py's recipe, KV cache pre-filled with random
rows) add the real LayerNorm, attention and GEMM shapes; there the mat-mul checks take the first and last row of each 128-row tile and
the last row (every token and every attention head is still checked)."""
import os
import numpy as np
import pytest
import pyoracle as po
import engine_nodes as en
from helpers import TINY_40B, TINY_7B, synth_model
from test_real_geometry_gpu import GEOM, MODEL_SEED, random_model

pytestmark = pytest.mark.gpu


def _kernel_of(t, K):
    import ggllm_cpp_b200.binding as b
    s = b.mmv_launch_shape(t, K)
    return ("generic",) if s is None else ("fast", s[0], s[1])


def read_tap(f, m, N, nr, layer_ids=None):
    """{node: array} per local layer (or per layer of layer_ids), the head's nodes and qkv_rotated per layer, of the most recent eval"""
    E, FF = m.E, m.FF
    act = {}
    for name in ("transformer.h.0.self_attention.query_key_value.weight", "lm_head.weight"):
        t = m.wtype(name)
        act[name] = po.VEC_DOT_TYPE.get(t)

    def actq_nodes(at, K, rows, pre):
        if at is None:
            return []
        blk = 256 if at == po.Q8_K else 32
        out = [(pre + ".q", np.int8, (rows, K)), (pre + ".d", np.float32, (rows, K // blk)),
               (pre + ".bs", np.int16, (rows, K // (16 if at == po.Q8_K else 32)))]
        return out + ([(pre + ".s", np.float32, (rows, K // 32))] if at == po.Q8_1 else [])

    at = act["transformer.h.0.self_attention.query_key_value.weight"]
    spec = [("inp", np.float32, (N, E)), ("qkv", np.float32, (N, m.QKV)), ("att", np.float32, (N, E)), ("up", np.float32, (N, FF)),
            ("dn", np.float32, (N, E)), ("ao", np.float32, (N, E)), ("xh_a", np.float16, (N, E)), ("xh_b", np.float16, (N, FF)),
            ("xh_m", np.float16, (N, E)), ("gen_na", np.float32, (N, E)), ("gen_nm", np.float32, (N, E))]
    for pre, K in (("xa", E), ("xm", E), ("xatt", E), ("xup", FF)):
        spec += actq_nodes(at, K, N, pre)
    layers, rotated = [], []
    for l in range(m.hp["n_layer"]) if layer_ids is None else layer_ids:
        nd = {}
        for name, dt, shape in spec:
            try:
                nd[name] = f.tap_read(l, name, dt, shape)
            except KeyError:
                pass
        layers.append(nd)
        rotated.append(int(f.tap_read(l, "qkv_rotated", np.int32, (1,))[0]))
    head = {}
    hspec = [("inp", np.float32, (N, E)), ("gen_na", np.float32, (nr, E)), ("logits", np.float32, (nr, m.V))]
    hspec += actq_nodes(act["lm_head.weight"], E, nr, "xf")
    for name, dt, shape in hspec:
        try:
            head[name] = f.tap_read(-1, name, dt, shape)
        except KeyError:
            pass
    return layers, head, rotated


def kv_all(f, n_layer, n_ctx):
    return [f.kv_read(l, 0, n_ctx) for l in range(n_layer)]


def run(gpu, f, step, n_ctx_rope):
    """one eval: ("eval", tokens, n_past, all_logits) through b200_falcon_eval (decode: the captured graph), or ("eager", token, n_past)
    through b200_falcon_decode_dev with B200_NO_GRAPH (the same step enqueued eagerly).  -> (logits returned, head's first row)"""
    kind, toks, n_past = step[:3]
    toks = np.asarray(toks, np.int32)
    if kind == "eval":
        all_logits = step[3]
        return f.eval(toks, n_past, n_ctx_rope, all_logits=all_logits), 0 if all_logits else toks.size - 1
    L = gpu.lib()
    tok = gpu.DevBuf(src=toks)
    os.environ["B200_NO_GRAPH"] = "1"
    try:
        f.decode_dev(tok.ptr, n_past, n_ctx_rope)
    finally:
        del os.environ["B200_NO_GRAPH"]
    L.b200_stream_synchronize(f.stream())
    out = np.empty((1, f.n_vocab), np.float32)
    L.b200_memcpy_d2h(out.ctypes.data, f.logits_dev(), out.nbytes)
    return out, 0


def check_case(gpu, hp, tensors, n_ctx, n_batch, steps, kv_seed, n_ctx_rope=0, subset=False):
    """fills every KV row with random values (seed kv_seed), runs `steps` tap off, restores the KV cache, runs them tap on and checks
    every eval node by node"""
    m = en.Model(hp, tensors)
    f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch)
    f.set_tensors(tensors)
    NL = hp["n_layer"]
    rng = np.random.default_rng(kv_seed)
    w = m.HKV * m.D
    for l in range(NL):
        f.kv_write(l, 0, rng.standard_normal((n_ctx, w)).astype(np.float32), rng.standard_normal((n_ctx, w)).astype(np.float32))
    start = kv_all(f, NL, n_ctx)
    off = [run(gpu, f, s, n_ctx_rope)[0] for s in steps]
    kv_off = kv_all(f, NL, n_ctx)
    for l, (k, v) in enumerate(start):
        f.kv_write(l, 0, k, v)
    shadow = n_batch > 8 and m.D == 64
    theta = po.orc().theta_scale(m.D, n_ctx_rope or n_ctx)
    long_from = int(os.environ.get("B200_ATTN_LONG_FROM", "1024"))
    f.tap(True)
    try:
        before = start
        for i, s in enumerate(steps):
            logits, r0 = run(gpu, f, s, n_ctx_rope)
            toks, n_past = np.atleast_1d(np.asarray(s[1], np.int32)), s[2]
            N = toks.size
            # (h): the tap changes nothing the eval computes
            assert np.array_equal(logits.view(np.uint32), off[i].view(np.uint32)), "step %d: logits differ with the tap on" % i
            after = kv_all(f, NL, n_ctx)
            layers, head, rotated = read_tap(f, m, N, N - r0)
            sh = [f.kv_shadow_read(l, 0, n_past + N) for l in range(NL)] if shadow else None
            ev = en.Eval(toks, n_past, r0, before, after, sh, logits, theta, _kernel_of,
                         en.attention_kind(N, n_past, shadow, long_from=long_from), rows_subset=subset)
            en.check_eval(m, ev, layers, head, rotated)
            before = after
        for (k0, v0), (k1, v1) in zip(kv_off, before):
            assert np.array_equal(k0.view(np.uint32), k1.view(np.uint32)) and np.array_equal(v0.view(np.uint32), v1.view(np.uint32)), \
                "KV cache differs with the tap on"
    finally:
        f.tap(False)
        f.free()


# ------------------------------------------------------------------------------------------------ tiny models
MODELS = {"40b-q4_K": (TINY_40B, po.Q4_K, {}), "7b-q4_0": (TINY_7B, po.Q4_0, {}), "40b-q3_K": (TINY_40B, po.Q3_K, {}),
          "40b-q6_K": (TINY_40B, po.Q6_K, {}), "7b-q5_1": (TINY_7B, po.Q5_1, {}), "40b-f16": (TINY_40B, po.F16, {}),
          "40b-mixed": (TINY_40B, po.Q4_K, {"dense_4h_to_h": po.Q6_K, "query_key_value": po.Q5_0, "lm_head": po.Q8_0}),
          "7b-f16-lm_head": (TINY_7B, po.Q4_0, {"lm_head": po.F16})}
PROMPT = [11, 100, 101, 102, 103, 104, 105, 106, 107, 108]
# mode: (n_ctx, n_batch, steps, environment); the KV rows before n_past hold random values
MODES = {"prompt8": (64, 8, [("eval", PROMPT[:8], 3, True)], {}),
         "prompt40": (128, 64, [("eval", list(range(12, 52)), 5, True)], {}),
         "decode": (64, 8, [("eval", [200], 6, False), ("eval", [203], 7, False), ("eager", [206], 8)], {}),
         "decode_no_fused": (64, 8, [("eval", [200], 6, False), ("eval", [203], 7, False)], {"B200_NO_FUSED_DECODE": "1"}),
         "decode_long_tier": (64, 8, [("eval", [200 + i], 10 + i, False) for i in range(4)], {"B200_ATTN_LONG_FROM": "12"})}
_tensors = {}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("model", list(MODELS))
def test_engine_nodes_tiny(gpu, monkeypatch, model, mode):
    hp, wt, overrides = MODELS[model]
    if model not in _tensors:
        _tensors[model] = synth_model(hp, wt, seed=1234, overrides=overrides)
    n_ctx, n_batch, steps, env = MODES[mode]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    long0 = gpu.lib().b200_attention_long_launches()
    check_case(gpu, hp, _tensors[model], n_ctx, n_batch, steps, kv_seed=7)
    if mode == "decode_long_tier":
        assert gpu.lib().b200_attention_long_launches() > long0                  # the long tier was really taken


# ------------------------------------------------------------------------------------------------ real widths
N_CTX = 8192


@pytest.mark.parametrize("geom,wtype,n_batch,steps", [
    ("40b", po.Q4_K, 512, [("eval", [17], 2040, False), ("eval", [18], 8184, False),
                           ("eval", (np.arange(96) * 7 + 13) % 2048, 2048 - 96, False),
                           ("eval", (np.arange(512) * 5 + 3) % 2048, 1536, False)]),
    ("7b", po.Q4_0, 8, [("eval", [317], 300, False)]),
    ("180b", po.Q4_K, 8, [("eval", [17], 0, False)]),
])
def test_engine_nodes_real_geometry(gpu, geom, wtype, n_batch, steps):
    """decode for 40B Q4_K at n_past 2040 and 8184, 7B Q4_0 at 300, 180B Q4_K at 0; a 96-token prompt chunk ending at 2048 and one
    512-token chunk (two 256-token GEMM tiles) of the 40B geometry"""
    hp = GEOM[geom]
    tensors = random_model(hp, wtype, seed=MODEL_SEED[geom] + wtype)
    check_case(gpu, hp, tensors, N_CTX, n_batch, steps, kv_seed=99, n_ctx_rope=N_CTX, subset=True)
