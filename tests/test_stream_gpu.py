"""-m gpu: streamed layers (b200_falcon_create_streamed, binding.Falcon(streamed=...)).

A streamed layer keeps its four matrices in pinned host memory and every eval copies them into one of two device slots before the layer
runs; the kernels read the same bytes from HBM as for a resident layer.  So every case below builds a resident engine and a streamed
engine from the same tensors and requires BIT-IDENTICAL results: logits, KV cache rows, sampled ids, scores, embeddings and tapped nodes.
"""
import ctypes as C
import functools
import importlib.util
import os

import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model, ggcc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

H40, H7 = dict(TINY_40B, n_layer=4), dict(TINY_7B, n_layer=4)
# name -> (hparams, weight type, overrides): fused decode + tensor-core prompt (Q4_K, Q4_0, Q3_K), the two-stream path with the generic
# mat-vec (Q6_K), the generic path (one layer in F16, an unquantised model)
MODELS = {
    "40b_q4_k": (H40, po.Q4_K, None), "7b_q4_0": (H7, po.Q4_0, None), "40b_q3_k": (H40, po.Q3_K, None), "40b_q6_k": (H40, po.Q6_K, None),
    "7b_mixed": (H7, po.Q4_0, {"h.1.": po.F16}), "40b_f16": (H40, po.F16, None),
}
SETS = {"first": [0], "last": [3], "gaps": [0, 2], "all": [0, 1, 2, 3]}
N_CTX, N_BATCH = 96, 48


@functools.lru_cache(maxsize=None)
def tensors(name, seed=1234):
    hp, wt, ov = MODELS[name]
    return synth_model(hp, wt, seed=seed, overrides=ov)


def engine(gpu, name, streamed=(), kv_f16=False, load="set", path=None, n_ctx=N_CTX, n_batch=N_BATCH):
    hp, wt, _ = MODELS[name]
    f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch, kv_f16=kv_f16, streamed=streamed)
    if load == "set":
        f.set_tensors(tensors(name))
    elif load == "random":
        f.set_random(ggcc.falcon_shapes(hp), wt, seed=5)
    else:
        f.load_ggcc(path)
    return f


def session(gpu, f, hp):
    """every evaluating call of part B in one fixed order, decode graphs on both sides of the long-context tier -> [(what, array)]"""
    out = []
    V = hp["n_vocab"]
    p5, p40 = np.array([11, 100, 101, 102, 103], np.int32), (np.arange(40, dtype=np.int32) * 37 + 5) % V
    out.append(("eval 5 all", f.eval(p5, 0, all_logits=True)))
    out.append(("eval 1 host graph tier 0", f.eval(np.array([104], np.int32), 5)))
    out.append(("eval 40", f.eval(p40, 6)))
    out.append(("eval 40 all", f.eval(p40[:8], 46, all_logits=True)))
    out.append(("eval 1 host graph tier 1", f.eval(np.array([7], np.int32), 54)))
    tok = gpu.DevBuf(src=np.array([9], np.int32))
    f.decode_dev(tok.ptr, 55)
    out.append(("decode_dev tier 1", _dev_logits(gpu, f, V)))
    f.decode_dev(tok.ptr, 4)
    out.append(("decode_dev tier 0", _dev_logits(gpu, f, V)))
    for l in range(hp["n_layer"]):
        k, v = f.kv_read(l, 0, 56)
        out += [("kv k %d" % l, k), ("kv v %d" % l, v)]
    f.eval(p5, 0)
    out.append(("generate_greedy", f.generate_greedy(104, 5, 12)))           # crosses the tier at 12 keys
    f.eval(p5, 0)
    out.append(("generate_chain", f.generate_chain(gpu.SamplingChain(top_k=20, temp=0.9, seed=3), [11, 100], 104, 5, 12)))
    out.append(("score", f.score(p40[:20], 0, np.r_[p40[1:20], -1].astype(np.int32))))
    ppl, nll = f.perplexity(np.r_[p40, p40].astype(np.int32), 32)
    out += [("perplexity", ppl), ("perplexity terms", nll)]
    f.set_embeddings(True)
    out.append(("embeddings logits", f.eval(p5, 0)))
    out.append(("embeddings", f.embeddings()))
    f.set_embeddings(False)
    return out


def _dev_logits(gpu, f, V):
    L = gpu.lib()
    L.b200_stream_synchronize(f.stream())
    out = np.empty(V, np.float32)
    L.b200_memcpy_d2h(gpu._np_ptr(out), f.logits_dev(), out.nbytes)
    return out


def assert_same(a, b):
    assert len(a) == len(b)
    for (wa, xa), (wb, xb) in zip(a, b):
        assert wa == wb
        np.testing.assert_array_equal(xa, xb, err_msg=wa)


@functools.lru_cache(maxsize=None)
def resident_session(gpu, name, kv_f16=False, load="set"):
    f = engine(gpu, name, kv_f16=kv_f16, load=load)
    out = session(gpu, f, MODELS[name][0])
    f.free()
    return out


@pytest.fixture
def long_tier(monkeypatch):
    monkeypatch.setenv("B200_ATTN_LONG_FROM", "12")


@pytest.mark.parametrize("which", list(SETS))
@pytest.mark.parametrize("name", list(MODELS))
def test_streamed_engine_equals_resident(gpu, long_tier, name, which):
    f = engine(gpu, name, streamed=SETS[which])
    assert f.stream_info()["layers"] == SETS[which]
    assert_same(session(gpu, f, MODELS[name][0]), resident_session(gpu, name))
    f.free()


@pytest.mark.parametrize("name,which", [("40b_q4_k", "gaps"), ("7b_q4_0", "all")])
def test_streamed_engine_fp16_kv(gpu, long_tier, name, which):
    f = engine(gpu, name, streamed=SETS[which], kv_f16=True)
    assert_same(session(gpu, f, MODELS[name][0]), resident_session(gpu, name, kv_f16=True))
    f.free()


@pytest.mark.parametrize("name", ["40b_q4_k", "40b_q6_k"])
def test_streamed_engine_random_tensors(gpu, long_tier, name):
    """set_tensor_random builds a streamed matrix in its slot from the same seed and index: the same bytes"""
    f = engine(gpu, name, streamed=SETS["gaps"], load="random")
    assert_same(session(gpu, f, MODELS[name][0]), resident_session(gpu, name, load="random"))
    f.free()


@pytest.mark.parametrize("name", ["40b_q4_k", "7b_mixed", "40b_f16"])
def test_streamed_engine_loads_ggcc(gpu, long_tier, name, tmp_path):
    """load_ggcc takes streamed matrices through a slot (staged rows, the device repack, D2H into the image); F16 matrices through set_tensor"""
    hp, wt, _ = MODELS[name]
    path = str(tmp_path / "m.ggcc")
    ggcc.write_ggcc(path, hp, tensors(name), ftype=ggcc.FTYPE_OF_TYPE.get(wt, 0))
    f = engine(gpu, name, streamed=SETS["gaps"], load="ggcc", path=path)
    assert_same(session(gpu, f, hp), resident_session(gpu, name))
    f.free()


@pytest.mark.parametrize("name", ["40b_q4_k", "7b_mixed"])
def test_tap_nodes_of_a_streamed_layer(gpu, name):
    hp = MODELS[name][0]
    E, QKV = hp["n_embd"], (hp["n_head"] + 2 * hp["n_head_kv"]) * (hp["n_embd"] // hp["n_head"])
    got = []
    for streamed in ((), [2]):
        f = engine(gpu, name, streamed=streamed)
        f.tap_layers([2])
        rows = []
        for toks, pos in ((np.array([11, 100, 101, 102, 103, 104, 105, 106, 107, 108], np.int32), 0), (np.array([7], np.int32), 10)):
            f.eval(toks, pos)
            n = toks.size
            rows += [f.tap_read(2, node, np.float32, (n, w)) for node, w in (("inp", E), ("qkv", QKV), ("att", E), ("up", 4 * E), ("dn", E), ("ao", E))]
            rows.append(f.tap_read(-1, "logits", np.float32, (1, hp["n_vocab"])))
        got.append(rows)
        f.free()
    for a, b in zip(*got):
        np.testing.assert_array_equal(a, b)


def test_replacing_a_streamed_matrix_after_its_graphs_exist(gpu):
    """a new wo for a streamed layer reaches its host image: the result changes, and equals a resident engine given the same wo.  A new
    type for a streamed matrix resizes the slots (the graphs are rebuilt around them)"""
    name = "40b_q4_k"
    hp = MODELS[name][0]
    other = synth_model(hp, po.Q4_K, seed=99)
    wo, up = "transformer.h.2.self_attention.dense.weight", "transformer.h.2.mlp.dense_h_to_4h.weight"
    res, st = engine(gpu, name), engine(gpu, name, streamed=[0, 2])
    p5, t = np.array([11, 100, 101, 102, 103], np.int32), np.array([104], np.int32)
    tok = gpu.DevBuf(src=np.array([9], np.int32))

    def step(f):
        f.eval(p5, 0)
        a = f.eval(t, 5)
        f.decode_dev(tok.ptr, 6)
        return a, _dev_logits(gpu, f, hp["n_vocab"])

    before = [step(f) for f in (res, st)]
    for f in (res, st):
        f.set_tensor(wo, *other[wo])
    after = [step(f) for f in (res, st)]
    for x, y in zip(*after):
        np.testing.assert_array_equal(x, y)
    assert not np.array_equal(after[1][0], before[1][0]) and not np.array_equal(after[1][1], before[1][1])
    slots = st.stream_info()["slot_bytes"]
    up8 = po.orc().quantize(po.Q8_0, synth_model(hp, po.F32, seed=1234)[up][2])      # the same weights as Q8_0
    for f in (res, st):
        f.set_tensor(up, po.Q8_0, tensors(name)[up][1], up8)
    info = st.stream_info()
    assert info["slot_bytes"] > slots
    assert info["copy_bytes"] == info["host_bytes"] == layer_bytes(hp, [po.Q4_K] * 4) + layer_bytes(hp, [po.Q4_K, po.Q4_K, po.Q8_0, po.Q4_K])
    changed = [step(f) for f in (res, st)]
    for x, y in zip(*changed):
        np.testing.assert_array_equal(x, y)
    res.free(); st.free()


@functools.lru_cache(maxsize=1)
def plan():
    spec = importlib.util.spec_from_file_location("stream_bench", os.path.join(ROOT, "tools", "stream_bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def layer_bytes(hp, types):
    sb = plan()
    return sum(sb.matrix_image_bytes(t, K, M) for t, (K, M) in zip(types, sb.layer_shapes(hp)))


def test_refusals(gpu):
    L = gpu.lib()
    hp = H40

    def create(streamed, kv=0, world=1, last=4):
        p = gpu.FalconParams(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["falcon_type"], 64, 8, 0, last, 0, world)
        a = np.ascontiguousarray(streamed, dtype=np.int32)
        return L.b200_falcon_create_streamed(C.byref(p), kv, gpu._np_ptr(a), a.size)

    assert not create([4]) and not create([-1]) and not create([2], last=2)          # outside [layer_first, layer_last)
    assert not create([1, 1]) and not create([0, 2, 0])                             # repeated
    assert not create([1], kv=2) and not create([1], kv=8)                          # not an f32 / f16 cache
    assert not create([0], world=2, last=2)                                         # a pipeline rank
    h = create([])
    assert h and L.b200_falcon_stream_info(h, None, None, None, None) == 0
    L.b200_falcon_free(h)
    h = create([3, 1])
    ids = np.zeros(2, np.int32)
    assert h and L.b200_falcon_stream_info(h, gpu._np_ptr(ids), None, None, None) == 2 and list(ids) == [1, 3]
    L.b200_falcon_free(h)
    with pytest.raises(ValueError):
        gpu.Falcon(hp, n_ctx=64, streamed=[7])


def _mem_used():
    rt = C.CDLL("libcudart.so.12")
    free, total = C.c_size_t(0), C.c_size_t(0)
    assert rt.cudaMemGetInfo(C.byref(free), C.byref(total)) == 0
    return total.value - free.value


def test_stream_info_and_device_memory(gpu):
    """stream_info reports the bytes wplanes_layout gives; the device holds two slots instead of the streamed layers"""
    hp = dict(n_vocab=1024, n_embd=2048, n_head=32, n_head_kv=4, n_layer=6, falcon_type=40)
    shapes = ggcc.falcon_shapes(hp)
    lay = layer_bytes(hp, [po.Q4_K] * 4)
    used = []
    for streamed in ((), [1, 2, 3, 4, 5]):
        gpu.lib().b200_synchronize()
        u0 = _mem_used()
        f = gpu.Falcon(hp, n_ctx=64, n_batch=1, streamed=streamed)
        f.set_random(shapes, po.Q4_K, seed=3)
        f.eval(np.array([1], np.int32), 0)
        used.append(_mem_used() - u0)
        info = f.stream_info()
        assert info["layers"] == list(streamed)
        n = len(streamed)
        assert info["copy_bytes"] == info["host_bytes"] == n * lay
        assert info["slot_bytes"] == (2 * lay if n else 0)
        f.free()
    assert used[0] - used[1] >= 3 * lay, (used, lay)


def test_falcon_40b_widths_one_streamed_layer(gpu):
    """real widths: Falcon-40B with 3 layers, the middle one streamed, random Q4_K weights; decode (both graphs) and a 512-token prompt"""
    hp = dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=3, falcon_type=40)
    shapes = ggcc.falcon_shapes(hp)
    outs = []
    for streamed in ((), [1]):
        f = gpu.Falcon(hp, n_ctx=1024, n_batch=512, streamed=streamed)
        f.set_random(shapes, po.Q4_K, seed=11)
        toks = (np.arange(512, dtype=np.int32) * 7919) % hp["n_vocab"]
        o = [f.eval(toks, 0, all_logits=True)[::37], f.eval(np.array([5], np.int32), 512)]
        tok = gpu.DevBuf(src=np.array([9], np.int32))
        f.decode_dev(tok.ptr, 513)
        o.append(_dev_logits(gpu, f, hp["n_vocab"]))
        o += list(f.kv_read(1, 500, 14))
        outs.append(o)
        f.free()
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)
