"""-m gpu: the fp16 KV cache (b200_falcon_create_kv with GGML_TYPE_F16, binding.Falcon(kv_f16=True)).

  * kernels, through the _kv16 hooks: every attention reader over an fp16 cache -- split-KV decode in the short and the long tier,
    the single-kernel decode (B200_ATTN_NOSPLIT), the CUDA-core prompt kernels (B200_ATTN_SIMT) and the wgmma prompt kernel -- held
    to tests/attn_exact.py's bound for its tier, computed on the widened cache the device holds afterwards; the appended K row is
    f16 of b200_rope_neox's rotation bit for bit, the V row f16(v), rows past T untouched
  * prompt identity: the wgmma prompt kernel reads only the fp16 planes, so an fp16 and an f32 engine give bit-identical logits over
    chunks of more than 8 tokens, and the fp16 engine's cache equals the f32 engine's fp16 copy bit for bit
  * engine: prompt, decode across both tiers, greedy generation and graph replay against the oracle with an fp16 cache
    (tests/kv16_twin.py), within test_falcon_gpu.py's tolerances
  * cache rows past the causal limit (NaN, or 1e6 = Inf in fp16) reach neither logits nor appended rows
  * state: kv_write / kv_read round and widen, save_kv / load_kv across both engine types, kv_fill_random, and the API edges
"""
import ctypes as C
import numpy as np
import pytest
import pyoracle as po
import attn_exact as ax
from helpers import TINY_40B, TINY_7B, synth_model
from kv16_twin import Kv16Twin
from test_attention_exact_gpu import MODES, HD, _inputs, _check
from test_falcon_gpu import assert_logits_close, assert_mostly_tight

pytestmark = pytest.mark.gpu


def h16(x):
    """f32 rows -> fp16 bit patterns (round to nearest even)"""
    return np.ascontiguousarray(np.asarray(x, np.float32).astype(np.float16).view(np.uint16))


def w16(b):
    """fp16 bit patterns -> exactly widened f32"""
    return np.asarray(b, np.uint16).view(np.float16).astype(np.float32)


# (G, n_head_kv, n_tok, n_past): T = 127, 128, 256, 257, 2049 -- partial and full 64 / 128-key tiles, 9 .. 512 tokens
PROMPT_SHAPES = [(2, 3, 9, 118), (29, 2, 9, 119), (16, 2, 64, 191), (71, 1, 130, 126), (16, 1, 512, 1537), (16, 2, 5, 250)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("G,n_head_kv,n_tok,n_past", PROMPT_SHAPES)
@pytest.mark.parametrize("path", ["ws", "prefill"])
def test_prompt_attention_kv16_exact(gpu, orc, monkeypatch, path, G, n_head_kv, n_tok, n_past, mode):
    n_head, T = G * n_head_kv, n_past + n_tok
    n_ctx = T + 77
    qkv, kc, vc = _inputs(orc, mode, n_head, n_head_kv, n_tok, n_past, n_ctx, seed=T + G + MODES.index(mode))
    if path == "prefill":
        monkeypatch.setenv("B200_ATTN_SIMT", "1")
    elif n_tok <= 8:
        monkeypatch.setenv("B200_ATTN_TC", "1")
    k0, v0 = h16(kc), h16(vc)
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=k0), gpu.DevBuf(src=v0), gpu.DevBuf(n_tok * n_head * HD * 4)
    gpu.lib().b200_attention_kv16(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, HD, n_tok, n_past, n_ctx, n_ctx)
    got = od.download(np.float32, (n_tok, n_head, HD))
    rot = qd.download(np.float32, qkv.shape)                                                     # rotated in place
    K, V = kd.download(np.uint16, k0.shape), vd.download(np.uint16, v0.shape)
    assert np.array_equal(K[n_past:T].reshape(n_tok, -1), h16(rot[:, n_head * HD:(n_head + n_head_kv) * HD]))
    assert np.array_equal(V[n_past:T].reshape(n_tok, -1), h16(qkv[:, (n_head + n_head_kv) * HD:]))
    assert np.array_equal(K[:n_past], k0[:n_past]) and np.array_equal(K[T:], k0[T:]) and np.array_equal(V[T:], v0[T:])
    q = rot[:, :n_head * HD].reshape(n_tok, n_head, HD)
    out, bound = ax.reference(q, w16(K), w16(V), n_past, "ws" if path == "ws" else "fp32")
    _check(got, out, bound, "kv16 %s G %d T %d n_tok %d %s" % (path, G, T, n_tok, mode))


DECODE_SHAPES = [(2, 3, 127), (16, 2, 128), (29, 2, 129), (71, 1, 255), (2, 4, 256), (16, 1, 257), (29, 2, 2048), (71, 1, 2049)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("G,n_head_kv,T", DECODE_SHAPES)
@pytest.mark.parametrize("tier", ["short", "long", "nosplit"])
def test_decode_attention_kv16_exact(gpu, orc, monkeypatch, tier, G, n_head_kv, T, mode):
    """b200_attention_decode_kv16.  The new token's key is scored from its rounded value, as the cache holds it."""
    n_head, n_past = G * n_head_kv, T - 1
    n_ctx = T + 77
    QKV = (n_head + 2 * n_head_kv) * HD
    qkv, kc, vc = _inputs(orc, mode, n_head, n_head_kv, 1, n_past, n_ctx, seed=7 * T + G + MODES.index(mode))
    monkeypatch.setenv("B200_ATTN_LONG_FROM", "1" if tier == "long" else "1000000")
    if tier == "nosplit":
        monkeypatch.setenv("B200_ATTN_NOSPLIT", "1")
    long0 = gpu.lib().b200_attention_long_launches()
    k0, v0 = h16(kc), h16(vc)
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=k0), gpu.DevBuf(src=v0), gpu.DevBuf(n_head * HD * 4)
    gpu.lib().b200_attention_decode_kv16(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, HD, n_past, n_ctx, n_ctx, None)
    assert (gpu.lib().b200_attention_long_launches() > long0) == (tier == "long")
    got = od.download(np.float32, (1, n_head, HD))
    rd = gpu.DevBuf(src=qkv)
    gpu.lib().b200_rope_neox(rd.ptr, 1, n_head + n_head_kv, HD, QKV, n_past, n_ctx, 1, 2.0, 0)
    rot = rd.download(np.float32, (1, QKV))
    K, V = kd.download(np.uint16, k0.shape), vd.download(np.uint16, v0.shape)
    assert np.array_equal(K[n_past].reshape(-1), h16(rot[0, n_head * HD:(n_head + n_head_kv) * HD]))
    assert np.array_equal(V[n_past].reshape(-1), h16(qkv[0, (n_head + n_head_kv) * HD:]))
    assert np.array_equal(K[:n_past], k0[:n_past]) and np.array_equal(K[T:], k0[T:]) and np.array_equal(V[T:], v0[T:])
    q = rot[:, :n_head * HD].reshape(1, n_head, HD)
    out, bound = ax.reference(q, w16(K), w16(V), n_past, "long" if tier == "long" else "fp32")
    _check(got, out, bound, "kv16 decode %s G %d T %d %s" % (tier, G, T, mode))


@pytest.mark.parametrize("hp,wt", [(TINY_40B, po.Q4_K), (TINY_7B, po.Q4_0)])
def test_prompt_chunks_are_bit_identical_between_cache_types(gpu, hp, wt):
    """chunks of 23, 40, 64 and 9 tokens (> 8: the wgmma prompt kernel, which reads only the fp16 planes; partial 64-token tiles)"""
    hp, n_ctx = dict(hp), 200
    tensors = synth_model(hp, wt, seed=91)
    a, b = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=64), gpu.Falcon(hp, n_ctx=n_ctx, n_batch=64, kv_f16=True)
    for f in (a, b):
        f.set_tensors(tensors)
    assert (a.kv_type(), b.kv_type()) == (0, 1)
    n = 0
    for N in (23, 40, 64, 9):
        toks = (np.arange(N, dtype=np.int32) * 29 + n + 5) % hp["n_vocab"]
        la, lb = a.eval(toks, n, all_logits=True), b.eval(toks, n, all_logits=True)
        assert np.array_equal(la, lb), (N, float(np.abs(la - lb).max()))
        n += N
        for l in range(hp["n_layer"]):
            ka, vta = a.kv_shadow_read(l, 0, n)
            kb, vtb = b.kv_shadow_read(l, 0, n)
            assert np.array_equal(ka, kb) and np.array_equal(vta, vtb), (N, l)
            k, v = b.kv_read(l, 0, n)
            assert np.array_equal(h16(k).reshape(ka.shape), ka) and np.array_equal(h16(v).reshape(ka.shape).transpose(1, 2, 0), vta)
    a.free(); b.free()


@pytest.mark.parametrize("hp,wt", [(TINY_40B, po.Q4_K), (TINY_7B, po.Q4_0)])
def test_engine_matches_the_fp16_cache_oracle(gpu, orc, hp, wt, monkeypatch):
    """prompt (mat-vec batches of 8), decode across the long-context tier (threshold moved to 14 keys), greedy generation on the device
    against the host arg-max loop, graph replay twice with the same bits"""
    monkeypatch.setenv("B200_ATTN_LONG_FROM", "14")
    long0 = gpu.lib().b200_attention_long_launches()
    tensors = synth_model(hp, wt, seed=1234)
    n_ctx, n_batch = 64, 8
    f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch, kv_f16=True)
    f.set_tensors(tensors)
    o, o32 = Kv16Twin(orc, hp, tensors, n_ctx, kv_f16=True), po.OrcFalcon(hp, tensors, n_ctx=n_ctx)
    prompt = [11, 100, 101, 102, 103, 104, 105, 106, 107, 108, 109]
    outs = []
    for c0 in range(0, len(prompt), n_batch):
        chunk = np.array(prompt[c0:c0 + n_batch], np.int32)
        outs.append((f.eval(chunk, c0, all_logits=True), o.eval(chunk, c0, all_logits=True)))
        o32.eval(chunk, c0, all_logits=True)
    pos = len(prompt)
    for s in range(8):
        tok = np.array([200 + 3 * s], np.int32)
        outs.append((f.eval(tok, pos), o.eval(tok, pos)))
        d32 = np.abs(o32.eval(tok, pos) - outs[-1][1]).max()
        print("step %d: fp16-cache oracle vs f32-cache oracle max |diff| %.3g" % (s, d32))
        pos += 1
    assert_mostly_tight([assert_logits_close(got, want, "kv16 step %d" % i) for i, (got, want) in enumerate(outs)])
    assert gpu.lib().b200_attention_long_launches() > long0
    first = f.eval(np.array([33], np.int32), pos)                  # graph replay: the same position twice, the same bits
    assert np.array_equal(f.eval(np.array([33], np.int32), pos), first)
    start = np.array(prompt[:6], np.int32)
    tok0 = int(np.argmax(f.eval(start, 0)[0]))
    want, tok, p = [], tok0, len(start)
    for _ in range(12):
        tok = int(np.argmax(f.eval(np.array([tok], np.int32), p)[0])); want.append(tok); p += 1
    f.eval(start, 0)
    assert list(f.generate_greedy(tok0, len(start), 12)) == want
    f.free()


ENGINE_TIERS = {"decode_short": (37, 1), "decode_long": (100, 1), "chunk_prefill": (61, 5), "chunk_ws": (50, 12)}


@pytest.mark.parametrize("garbage", [np.nan, 1e6])
@pytest.mark.parametrize("tier", list(ENGINE_TIERS))
def test_kv16_engine_ignores_cache_rows_past_the_causal_limit(gpu, monkeypatch, tier, garbage):
    """two fp16 engines, one with NaN (or 1e6, which kv_write rounds to Inf) in every cache row from n_past on, one with zeros:
    bit-identical logits and appended rows"""
    n_past, N = ENGINE_TIERS[tier]
    hp, n_ctx = dict(TINY_40B), 200
    if tier == "decode_long":
        monkeypatch.setenv("B200_ATTN_LONG_FROM", "64")
    long0 = gpu.lib().b200_attention_long_launches()
    tensors = synth_model(hp, po.Q4_K, seed=61)
    rng = np.random.default_rng(62)
    w = hp["n_head_kv"] * HD
    engines = []
    for fill in (garbage, 0.0):
        f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16, kv_f16=True)
        f.set_tensors(tensors)
        engines.append(f)
    for l in range(hp["n_layer"]):
        k0, v0 = rng.standard_normal((n_past, w)).astype(np.float32), rng.standard_normal((n_past, w)).astype(np.float32)
        for f, fill in zip(engines, (garbage, 0.0)):
            pad = np.full((n_ctx - n_past, w), fill, np.float32)
            f.kv_write(l, 0, np.concatenate([k0, pad]), np.concatenate([v0, pad]))
    k_stale, _ = engines[0].kv_read(0, n_past + N, 1)
    assert (np.isnan(k_stale) if np.isnan(garbage) else np.isinf(k_stale)).all()
    toks = (np.arange(N, dtype=np.int32) * 37 + 11) % hp["n_vocab"]
    a, b = [f.eval(toks, n_past, all_logits=True) for f in engines]
    assert np.isfinite(b).all()
    assert np.array_equal(a, b), (tier, int(np.isnan(a).sum()))
    for l in range(hp["n_layer"]):
        ka, va = engines[0].kv_read(l, n_past, N)
        kb, vb = engines[1].kv_read(l, n_past, N)
        assert np.array_equal(ka, kb) and np.array_equal(va, vb)
    if tier == "decode_long":
        assert gpu.lib().b200_attention_long_launches() > long0
    for f in engines:
        f.free()


def test_kv16_state_round_trips(gpu, tmp_path):
    hp, n_ctx = dict(TINY_40B), 100
    w = hp["n_head_kv"] * HD
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((n_ctx, w)) * np.float32(3.0)).astype(np.float32)
    x[0, :4] = [70000.0, -1e9, 1e-8, 65519.0]                       # +Inf, -Inf, an fp16 subnormal, the largest value that rounds to 65504
    f16e = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16, kv_f16=True)
    f32e = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16)
    for l in range(hp["n_layer"]):
        f16e.kv_write(l, 0, x, -x)
        f32e.kv_write(l, 0, x, -x)
    k, v = f16e.kv_read(1, 0, n_ctx)
    assert np.array_equal(k, w16(h16(x))) and np.array_equal(v, w16(h16(-x)))
    assert k[0, 0] == np.inf and k[0, 1] == -np.inf and k[0, 3] == 65504.0
    # save / load: an fp16 engine's file round-trips bit for bit into either engine type; an f32 file is rounded by an fp16 engine
    p16, p32 = str(tmp_path / "a16.kv"), str(tmp_path / "a32.kv")
    f16e.save_kv(p16, n_ctx)
    f32e.save_kv(p32, n_ctx)
    g16 = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16, kv_f16=True)
    g32 = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16)
    for g, path, want in ((g16, p16, w16(h16(x))), (g32, p16, w16(h16(x))), (g16, p32, w16(h16(x))), (g32, p32, x)):
        assert g.load_kv(path) == n_ctx
        for l in range(hp["n_layer"]):
            k, v = g.kv_read(l, 0, n_ctx)
            assert np.array_equal(k, want) and np.array_equal(v, -want), (path, g.kv_type(), l)
    # kv_fill_random: the f32 engine's values, rounded
    f16e.kv_fill_random(10, 20, seed=3)
    f32e.kv_fill_random(10, 20, seed=3)
    for l in range(hp["n_layer"]):
        k16, v16 = f16e.kv_read(l, 10, 20)
        k32, v32 = f32e.kv_read(l, 10, 20)
        assert np.array_equal(k16, w16(h16(k32))) and np.array_equal(v16, w16(h16(v32)))
        kp, vt = f16e.kv_shadow_read(l, 10, 20)
        assert np.array_equal(kp.reshape(20, -1), h16(k16)) and np.array_equal(vt, h16(v16).reshape(20, -1, HD).transpose(1, 2, 0))
    for f in (f16e, f32e, g16, g32):
        f.free()


def test_kv16_api_edges(gpu):
    hp = dict(TINY_40B)
    L = gpu.lib()
    params = gpu.FalconParams(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["falcon_type"], 128, 1, 0, 2, 0, 1)
    for t in (-1, 2, 8, 12):
        assert not L.b200_falcon_create_kv(C.byref(params), t)
    NL, HKV = hp["n_layer"], hp["n_head_kv"]
    for n_ctx in (100, 128):
        pad = (n_ctx + 63) // 64 * 64
        got = {}
        for n_batch in (1, 512):
            for kv16 in (False, True):
                f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch, kv_f16=kv16)
                assert f.kv_type() == int(kv16)
                vt = n_batch > 8
                if kv16:
                    want = NL * pad * HKV * HD * 2 * (2 + vt)
                else:
                    want = NL * n_ctx * HKV * HD * 4 * 2 + vt * NL * pad * HKV * HD * 2 * 2
                assert f.kv_device_bytes() == want, (n_ctx, n_batch, kv16)
                got[n_batch, kv16] = want
                if kv16 and not vt:                                      # the K cache is the fp16 K plane; no V^T at n_batch <= 8
                    k = np.empty(HKV * HD, np.uint16)
                    assert L.b200_falcon_kv_shadow_read(f.h, 0, 0, 1, k.ctypes.data, None) == 0
                    assert L.b200_falcon_kv_shadow_read(f.h, 0, 0, 1, k.ctypes.data, k.ctypes.data) == 1
                f.free()
        if n_ctx % 64 == 0:
            for n_batch in (1, 512):
                assert 2 * got[n_batch, True] == got[n_batch, False]
