"""-m gpu: every attention kernel the engine can choose, held to the exact-arithmetic reference of tests/attn_exact.py within its
per-element bound, plus the two properties of the KV cache the kernels rely on.

  * kernels, through the C ABI: split-KV decode in the short tier (attention.cu) and in the long tier (attention_long.cu, selected by
    B200_ATTN_LONG_FROM), the CUDA-core prompt kernels (attention_prefill.cu, B200_ATTN_SIMT) and the wgmma prompt kernel
    (attention_ws.cu, B200_ATTN_TC below 9 tokens).  Shapes: G = 2 / 16 / 29 / 71 query heads per KV head, T = n_past + n_tok at
    128-key tile edges (127 .. 257, 2048, 2049), n_past not a multiple of 64, row counts G * n_tok that are not multiples of 128.
    The reference reads the device's own rotated rows (q from the rotated qkv buffer, k from the cache), so RoPE stays out of it.
  * inputs: random; "future" (keys past each query's causal limit aligned with it, V = 100 there: a leaked key takes most of the
    probability); "peaked" (the row maximum at key 0, at the last visible key, at the first / last key of a middle tile or in the
    partial last tile, scores from -50 to 30); "flat" (q = 0: the exact mean of V); "mag_lo" / "mag_hi" (V x 1e-3 with scores ~1e-2,
    V x 1e2 with scores up to ~50; every ws operand stays far below fp16's 65504)
  * engine: logits and appended K / V rows do not depend on cache rows past the causal limit (NaN, or 1e6 = Inf in the fp16 copy)
  * engine: the fp16 copy of the cache (k16, V^T) equals f16 of the fp32 cache bit for bit after every kind of write
"""
import numpy as np
import pytest
import pyoracle as po
import attn_exact as ax
from helpers import TINY_40B, TINY_7B, synth_model

pytestmark = pytest.mark.gpu
HD = 64
MODES = ("random", "future", "peaked", "flat", "mag_lo", "mag_hi")


def _inv_rope(orc, x, n_past, n_ctx):
    """R(-theta) x per NeoX pair (i, i + 32) at positions n_past + t: rows that the device's RoPE turns (up to rounding) into x"""
    y = np.array(x, np.float32)
    y[..., HD // 2:] *= -1
    y = orc.rope_neox(y, n_past, n_ctx)
    y[..., HD // 2:] *= -1
    return y


def _inputs(orc, mode, n_head, n_head_kv, n_tok, n_past, n_ctx, seed):
    """-> qkv [n_tok][(n_head + 2 n_head_kv) 64] (before RoPE), k / v cache [n_ctx][n_head_kv][64]: rows [0, n_past) hold the
    context, rows [T, n_ctx) stale values no kernel may read.  The post-RoPE q / k are designed; the new tokens' rows are
    pre-rotated backwards so that the device's rotation yields them."""
    rng = np.random.default_rng(seed)
    T = n_past + n_tok
    K = rng.standard_normal((n_ctx, n_head_kv, HD)).astype(np.float32)
    V = rng.standard_normal((n_ctx, n_head_kv, HD)).astype(np.float32)
    Q = rng.standard_normal((n_tok, n_head, HD)).astype(np.float32)
    pos = n_past + np.arange(n_tok)
    if mode == "future":
        # key j points along axis j % 64, query at position p along axis (p + 1) % 64: its first key past the causal limit (and every
        # 64th before it) scores 0.125 * 12 * 12 = 18, the rest ~0.  New-token and stale V rows carry the marker 100.
        K = 0.1 * K
        K[np.arange(n_ctx), :, np.arange(n_ctx) % HD] += 12.0
        Q = 0.1 * Q
        Q[np.arange(n_tok), :, (pos + 1) % HD] += 12.0
        V[n_past:] = 100.0 + 0.1 * V[n_past:]
    elif mode == "peaked":
        # five classes of rows, class c = (t + h) % 5 points along axis c; keys have components U(-20, 12) on the axes 0..4
        # (scores 0.125 * 20 * [-20, 12] = -50 .. 30), and the row maximum 0.125 * 20 * 20 = 50 sits at key 0 (class 0), at every new
        # key (class 1: the last visible key is one of them), at 128 and 255 (first / last key of the second tile), in the last tile
        K = 0.05 * K
        K[:, :, :5] = rng.uniform(-20.0, 12.0, (n_ctx, n_head_kv, 5))
        last = (T - 1) // 128 * 128 + ((T - 1) % 128) // 2
        for c, p in ((0, 0), (2, 128), (3, 255), (4, last)):
            if p < n_ctx:
                K[p, :, c] = 20.0
        K[n_past:T, :, 1] = 20.0
        Q = 0.05 * Q
        cls = (np.arange(n_tok)[:, None] + np.arange(n_head)[None, :]) % 5
        np.put_along_axis(Q, cls[:, :, None], np.take_along_axis(Q, cls[:, :, None], 2) + 20.0, 2)
    elif mode == "flat":
        Q[:] = 0.0
    elif mode == "mag_lo":
        Q, K, V = 0.1 * Q, 0.1 * K, 1e-3 * V
    elif mode == "mag_hi":
        Q, K, V = 4.0 * Q, 4.0 * K, 1e2 * V
    kc, vc = K.copy(), V.copy()
    kc[n_past:T] = 0.0
    vc[n_past:T] = 0.0
    qkv = np.concatenate([_inv_rope(orc, Q, n_past, n_ctx), _inv_rope(orc, K[n_past:T], n_past, n_ctx), V[n_past:T]], axis=1)
    return np.ascontiguousarray(qkv.reshape(n_tok, -1), np.float32), kc, vc


def _check(got, out, bound, what):
    r = np.abs(got.astype(np.float64) - out) / bound
    print("%s: max |err| / bound %.3g, max |err| %.3g, median |out| %.3g" % (what, r.max(), np.abs(got - out).max(), np.median(np.abs(out))))
    assert np.all(np.isfinite(got)), what
    assert r.max() <= 1.0, (what, float(r.max()), np.unravel_index(int(r.argmax()), r.shape))


# (G, n_head_kv, n_tok, n_past): T = 127, 128, 129, 255, 256, 257, 2048, 2049
PROMPT_SHAPES = [(2, 3, 9, 118), (29, 2, 9, 119), (71, 1, 9, 120), (16, 2, 64, 191), (71, 1, 130, 126), (29, 2, 130, 127),
                 (16, 1, 130, 1918), (16, 1, 512, 1537)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("G,n_head_kv,n_tok,n_past", PROMPT_SHAPES)
@pytest.mark.parametrize("path", ["ws", "prefill"])
def test_prompt_attention_exact(gpu, orc, monkeypatch, path, G, n_head_kv, n_tok, n_past, mode):
    n_head, T = G * n_head_kv, n_past + n_tok
    n_ctx = T + 77
    qkv, kc, vc = _inputs(orc, mode, n_head, n_head_kv, n_tok, n_past, n_ctx, seed=T + G + MODES.index(mode))
    if path == "prefill":
        monkeypatch.setenv("B200_ATTN_SIMT", "1")
    elif n_tok <= 8:
        monkeypatch.setenv("B200_ATTN_TC", "1")
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=kc), gpu.DevBuf(src=vc), gpu.DevBuf(n_tok * n_head * HD * 4)
    gpu.lib().b200_attention(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, HD, n_tok, n_past, n_ctx, n_ctx)
    got = od.download(np.float32, (n_tok, n_head, HD))
    q = qd.download(np.float32, qkv.shape)[:, :n_head * HD].reshape(n_tok, n_head, HD)      # rotated in place
    K, V = kd.download(np.float32, kc.shape), vd.download(np.float32, vc.shape)
    assert np.array_equal(V[n_past:T].reshape(n_tok, -1), qkv[:, (n_head + n_head_kv) * HD:])
    assert np.array_equal(K[T:], kc[T:]) and np.array_equal(V[T:], vc[T:])
    out, bound = ax.reference(q, K, V, n_past, "ws" if path == "ws" else "fp32")
    _check(got, out, bound, "%s G %d T %d n_tok %d %s" % (path, G, T, n_tok, mode))


# (G, n_head_kv, T): every G at every tile edge would be 32 shapes; each G meets two of them
DECODE_SHAPES = [(2, 3, 127), (16, 2, 128), (29, 2, 129), (71, 1, 255), (2, 4, 256), (16, 1, 257), (29, 2, 2048), (71, 1, 2049)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("G,n_head_kv,T", DECODE_SHAPES)
@pytest.mark.parametrize("tier", ["short", "long"])
def test_decode_attention_exact(gpu, orc, monkeypatch, tier, G, n_head_kv, T, mode):
    """b200_attention_decode (RoPE + append fused into the split-KV kernels).  Its q is rotated in registers: the test rotates a copy
    with b200_rope_neox, whose arithmetic is the same -- the copy's key row must equal the appended one bit for bit."""
    n_head, n_past = G * n_head_kv, T - 1
    n_ctx = T + 77
    QKV = (n_head + 2 * n_head_kv) * HD
    qkv, kc, vc = _inputs(orc, mode, n_head, n_head_kv, 1, n_past, n_ctx, seed=7 * T + G + MODES.index(mode))
    monkeypatch.setenv("B200_ATTN_LONG_FROM", "1" if tier == "long" else "1000000")
    long0 = gpu.lib().b200_attention_long_launches()
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=kc), gpu.DevBuf(src=vc), gpu.DevBuf(n_head * HD * 4)
    gpu.lib().b200_attention_decode(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, HD, n_past, n_ctx, n_ctx, None)
    assert (gpu.lib().b200_attention_long_launches() > long0) == (tier == "long")
    got = od.download(np.float32, (1, n_head, HD))
    rd = gpu.DevBuf(src=qkv)
    gpu.lib().b200_rope_neox(rd.ptr, 1, n_head + n_head_kv, HD, QKV, n_past, n_ctx, 1, 2.0, 0)
    rot = rd.download(np.float32, (1, QKV))
    K, V = kd.download(np.float32, kc.shape), vd.download(np.float32, vc.shape)
    assert np.array_equal(K[n_past].reshape(-1), rot[0, n_head * HD:(n_head + n_head_kv) * HD])
    assert np.array_equal(V[n_past].reshape(-1), qkv[0, (n_head + n_head_kv) * HD:])
    q = rot[:, :n_head * HD].reshape(1, n_head, HD)
    out, bound = ax.reference(q, K, V, n_past, "long" if tier == "long" else "fp32")
    _check(got, out, bound, "decode %s G %d T %d %s" % (tier, G, T, mode))


ENGINE_TIERS = {"decode_short": (37, 1), "decode_long": (100, 1), "chunk_prefill": (61, 5), "chunk_ws": (50, 12)}


@pytest.mark.parametrize("garbage", [np.nan, 1e6])
@pytest.mark.parametrize("tier", list(ENGINE_TIERS))
def test_engine_ignores_cache_rows_past_the_causal_limit(gpu, monkeypatch, tier, garbage):
    """two engines with the same model and context; in one, every cache row from n_past on holds NaN (or 1e6, Inf in the fp16 copy),
    in the other zeros.  The same tokens give bit-identical logits and appended K / V rows: a key past a query's causal limit must
    not reach any product, not even with probability 0 (0 x NaN = NaN).  chunk_ws: T = 62, inside the first 128-key tile."""
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
        f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16)
        f.set_tensors(tensors)
        engines.append(f)
    for l in range(hp["n_layer"]):
        k0, v0 = rng.standard_normal((n_past, w)).astype(np.float32), rng.standard_normal((n_past, w)).astype(np.float32)
        for f, fill in zip(engines, (garbage, 0.0)):
            pad = np.full((n_ctx - n_past, w), fill, np.float32)
            f.kv_write(l, 0, np.concatenate([k0, pad]), np.concatenate([v0, pad]))
    toks = (np.arange(N, dtype=np.int32) * 37 + 11) % hp["n_vocab"]
    a, b = [f.eval(toks, n_past, all_logits=True) for f in engines]
    assert np.isfinite(b).all()
    assert np.array_equal(a, b), (tier, int(np.isnan(a).sum()), float(np.nanmax(np.abs(a - b))) if np.isfinite(a).any() else None)
    for l in range(hp["n_layer"]):
        ka, va = engines[0].kv_read(l, n_past, N)
        kb, vb = engines[1].kv_read(l, n_past, N)
        assert np.array_equal(ka, kb) and np.array_equal(va, vb)
    if tier == "decode_long":
        assert gpu.lib().b200_attention_long_launches() > long0
    for f in engines:
        f.free()


def _check_shadow(f, n, n_ctx, what):
    """k16[p] == f16(k[p]) and V^T[:, :, p] == f16(v[p]) bit for bit for p < n; the padding columns [n_ctx, ctx_pad) are zero"""
    hkv = f.hp["n_head_kv"]
    ctx_pad = (n_ctx + 63) // 64 * 64
    for l in range(f.hp["n_layer"]):
        k, v = f.kv_read(l, 0, n)
        k16, vt16 = f.kv_shadow_read(l, 0, ctx_pad)
        assert np.array_equal(k16[:n], k.astype(np.float16).view(np.uint16).reshape(n, hkv, HD)), (what, l)
        assert np.array_equal(vt16[:, :, :n], v.astype(np.float16).view(np.uint16).reshape(n, hkv, HD).transpose(1, 2, 0)), (what, l)
        assert not k16[n_ctx:].any() and not vt16[:, :, n_ctx:].any(), (what, l)


@pytest.mark.parametrize("hp,env", [(TINY_40B, None), (TINY_7B, None), (TINY_40B, "B200_ATTN_NOSPLIT")])
def test_fp16_shadow_is_bit_exact_with_the_cache(gpu, monkeypatch, tmp_path, hp, env):
    """the fp16 copy the wgmma prompt kernel reads, after every writer: batched RoPE + append (2-8 and > 8 tokens, partial 64-token
    tiles of the V^T transpose at n_past 7 / 23 / 39 / 55 / 68), the fused decode appends of both tiers, greedy generation through
    the graph with a device n_past, kv_write into the middle, save_kv / load_kv into a fresh engine.  With B200_ATTN_NOSPLIT the
    decode steps append through the single-token RoPE + append kernel.  n_ctx = 200: the V^T rows are padded to 256."""
    if env:
        monkeypatch.setenv(env, "1")
    hp, n_ctx = dict(hp), 200
    tensors = synth_model(hp, po.Q4_K if hp["falcon_type"] == 40 else po.Q4_0, seed=71)
    f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16)
    f.set_tensors(tensors)
    toks = lambda n, s: (np.arange(n, dtype=np.int32) * 13 + s) % hp["n_vocab"]
    f.eval(toks(7, 3), 0)
    _check_shadow(f, 7, n_ctx, "7-token chunk")
    n = 7
    for N in (16, 16, 16, 13, 5):
        f.eval(toks(N, n), n)
        n += N
        _check_shadow(f, n, n_ctx, "%d-token chunk" % N)
    long0 = gpu.lib().b200_attention_long_launches()
    for i in range(2):
        f.eval(toks(1, n), n); n += 1
        _check_shadow(f, n, n_ctx, "decode step at %d" % (n - 1))
    monkeypatch.setenv("B200_ATTN_LONG_FROM", str(n + 2))
    for i in range(3):
        f.eval(toks(1, n), n); n += 1
        _check_shadow(f, n, n_ctx, "decode step at %d across the long tier" % (n - 1))
    assert gpu.lib().b200_attention_long_launches() > long0
    f.generate_greedy(11, n, 8)
    n += 8
    _check_shadow(f, n, n_ctx, "greedy generation")
    rng = np.random.default_rng(72)
    w = hp["n_head_kv"] * HD
    for l in range(hp["n_layer"]):
        f.kv_write(l, 30, rng.standard_normal((10, w)).astype(np.float32), rng.standard_normal((10, w)).astype(np.float32))
    _check_shadow(f, n, n_ctx, "kv_write")
    path = str(tmp_path / "s.kv")
    f.save_kv(path, n)
    g = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=16)
    assert g.load_kv(path) == n
    _check_shadow(g, n, n_ctx, "load_kv")
    with pytest.raises(RuntimeError):
        f.kv_shadow_read(0, 0, 257)
    with pytest.raises(RuntimeError):
        f.kv_shadow_read(hp["n_layer"], 0, 1)
    small = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=8)                     # no fp16 copy at n_batch <= 8
    with pytest.raises(RuntimeError):
        small.kv_shadow_read(0, 0, 1)
    f.free(); g.free(); small.free()
