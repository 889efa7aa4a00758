"""-m gpu: oracle parity at the head / width geometry of the models bench.py actually runs (Falcon-40B 8192/128/8,
Falcon-7B 4544/71/1, Falcon-180B 14848/232/8), not only at the tiny test shapes:

  * the 8-CTA thread-block-cluster LayerNorm (n_embd 8192), its 5-CTA ragged form (4544) and the two-pass register kernel (14848)
  * split-KV decode attention with G = 16 / 71 / 29 query heads per KV head, with and without the Q8 hand-over to `wo`,
    at n_past 0 / 300 / 2040 / 8184 of an 8192-token context
  * the wgmma prompt attention over 16 key tiles (T = 2048) and the wgmma GEMM at the real K
  * whole evals (2 layers, vocabulary 2048) through b200_falcon_eval at those positions

The 2-layer models carry well-formed pseudo-random blocks (ggcc.random_blocks: numpy-drawn blocks of the same kind as, but not the
bytes of, the device-made weights bench.py times -- those are tests/device_random.py's, checked in test_bench_models_gpu.py) and the
KV cache of BOTH the oracle and the engine is pre-filled with the same random rows (b200_falcon_kv_write), so a decode at
position 8184 attends over a full context without 8184 evals first.

Tolerance of the whole-eval comparisons: the "loose" bound of tests/test_falcon_gpu.py (max |diff| <= 2e-2 S, median <= 2e-3 S,
S = max |logit|) for EVERY eval.  The "tight" reassociation-level bound of the tiny models cannot hold at these widths for any pair of
implementations: one eval re-quantises ~57k activation values per layer to int8, ~1e-7 summation-order differences flip about one
code per layer per token, and each flip moves a mat-mul's outputs by ~3e-4 of their scale.  The reference's own AVX2 build and the
scalar oracle disagree by median 4e-4 .. 1.6e-3 S on exactly these models (tests/golden/real_geometry_cpu_vs_cpu.json, written by
tests/golden/make_real_geometry_yardstick.py) -- the same level the GPU is held to.  The per-operator tests below are the tight
ones: quantised codes bit-exact, fp32 attention to 2e-6.
"""
import os
import numpy as np
import pytest
import pyoracle as po
from helpers import ggcc
from test_falcon_gpu import assert_logits_close

pytestmark = pytest.mark.gpu

GEOM = {"40b": dict(n_vocab=2048, n_embd=8192, n_head=128, n_head_kv=8, n_layer=2, falcon_type=40),
        "7b": dict(n_vocab=2048, n_embd=4544, n_head=71, n_head_kv=1, n_layer=2, falcon_type=7),
        "180b": dict(n_vocab=2048, n_embd=14848, n_head=232, n_head_kv=8, n_layer=2, falcon_type=40)}
NTHREADS = max(8, min(os.cpu_count() or 8, 64))
MODEL_SEED = {"40b": 100, "7b": 200, "180b": 300}
N_CTX = 8192


def random_model(hp, wtype, seed):
    rng = np.random.default_rng(seed)
    tensors = {}
    for name, ne in ggcc.falcon_shapes(hp).items():
        if len(ne) == 1:
            v = (1.0 + 0.1 * rng.standard_normal(ne[0])) if name.endswith(".weight") else 0.01 * rng.standard_normal(ne[0])
            tensors[name] = (po.F32, ne, v.astype(np.float32))
        else:
            tensors[name] = (wtype, ne, ggcc.random_blocks(wtype, ne[1], ne[0], rng))
    return tensors


_models = {}


def model_pair(gpu, geom, wtype, n_batch):
    """(engine, oracle) over the same random model with the same random KV rows in every position; cached per module run"""
    key = (geom, wtype)
    if key in _models:
        return _models[key]
    for k in list(_models):                       # one resident pair at a time: the 180B-geometry one is ~1.3 GB on each side
        f, o = _models.pop(k)
        f.free()
    hp = GEOM[geom]
    tensors = random_model(hp, wtype, seed=MODEL_SEED[geom] + wtype)
    f = gpu.Falcon(hp, n_ctx=N_CTX, n_batch=n_batch)
    f.set_tensors(tensors)
    o = po.OrcFalcon(hp, tensors, n_ctx=N_CTX)
    rng = np.random.default_rng(99)
    for l in range(hp["n_layer"]):
        o.k[l] = rng.standard_normal(o.k[l].shape).astype(np.float32)
        o.v[l] = rng.standard_normal(o.v[l].shape).astype(np.float32)
        f.kv_write(l, 0, o.k[l], o.v[l])
        k2, v2 = f.kv_read(l, 4000, 7)
        assert np.array_equal(k2, o.k[l][4000:4007]) and np.array_equal(v2, o.v[l][4000:4007])
    _models[key] = (f, o)
    return f, o


@pytest.mark.parametrize("geom,wtype", [("40b", po.Q4_K), ("40b", po.Q3_K), ("7b", po.Q4_0), ("180b", po.Q4_K)])
def test_decode_at_real_geometry(gpu, geom, wtype):
    """b200_falcon_eval(n_tokens = 1) == oracle at n_past 0 / 300 / 2040 / 8184: the default decode graph of each model family
    (fused single-stream path for Q4_K / Q4_0, two-stream per-node path for Q3_K) with its real LayerNorm and attention shapes"""
    f, o = model_pair(gpu, geom, wtype, n_batch=96)
    for n_past in (0, 300, 2040, 8184):
        tok = np.array([17 + n_past % 1000], np.int32)
        got, want = f.eval(tok, n_past, N_CTX), o.eval(tok, n_past, N_CTX, nthreads=NTHREADS)
        assert_logits_close(got, want, "%s %s n_past %d" % (geom, po.TYPE_NAMES[wtype], n_past))
        # the K / V rows the step appended are the oracle's (RoPE at this position with the NTK alpha of n_ctx 8192)
        for l in range(GEOM[geom]["n_layer"]):
            k, v = f.kv_read(l, n_past, 1)
            assert np.allclose(k, o.k[l][n_past:n_past + 1], rtol=0, atol=2e-2 * np.abs(o.k[l][n_past]).max())
            assert np.allclose(v, o.v[l][n_past:n_past + 1], rtol=0, atol=2e-2 * np.abs(o.v[l][n_past]).max())


def test_prompt_chunk_at_real_geometry(gpu):
    """a 96-token chunk ending at position 2048 of the Falcon-40B geometry: wgmma GEMMs at K = 8192 / 32768 and wgmma attention over
    16 key tiles (T = 2048), against the oracle.  Tolerance: the GEMM-path bound of tests/test_falcon_gpu.py (fp16 operands)."""
    f, o = model_pair(gpu, "40b", po.Q4_K, n_batch=96)
    toks = (np.arange(96, dtype=np.int32) * 7 + 13) % 2048
    n_past = 2048 - 96
    got = f.eval(toks, n_past, N_CTX, all_logits=True)
    want = o.eval(toks, n_past, N_CTX, all_logits=True, nthreads=NTHREADS)
    scale = float(np.abs(want).max())
    d = np.abs(got - want)
    assert d.max() <= 3e-2 * scale and np.median(d) <= 5e-3 * scale, (float(d.max()), float(np.median(d)), scale)


@pytest.mark.parametrize("n,wtype,dual", [(8192, po.Q4_K, True), (8192, po.Q4_0, False), (4544, po.Q4_0, False), (14848, po.Q4_K, True), (2048, po.Q4_K, True)])
def test_layernorm_q_node(gpu, orc, n, wtype, dual):
    """the decode step's residual-add + LayerNorm(s) + Q8 quantisation node (cluster kernel: 8 CTAs at 8192, 5 ragged at 4544, 2 at 2048;
    register kernel at 14848): the residual row is exact and the quantised codes / scales / block sums are BIT-EXACT with
    quantize_row_q8_K / q8_0 applied to the oracle's LayerNorm of the same row (ggml.c:10540-10599, k_quants.c:899-934, ggml.c:1201-1237)"""
    rng = np.random.default_rng(n + wtype)
    x, ra, rb = [(s * rng.standard_normal(n)).astype(np.float32) for s in (1.0, 0.3, 0.2)]
    g1, g2 = [(1.0 + 0.1 * rng.standard_normal(n)).astype(np.float32) for _ in range(2)]
    b1, b2 = [(0.01 * rng.standard_normal(n)).astype(np.float32) for _ in range(2)]
    xd, rad, rbd = gpu.DevBuf(src=x), gpu.DevBuf(src=ra), gpu.DevBuf(src=rb)
    gd = [gpu.DevBuf(src=v) for v in (g1, b1, g2, b2)]
    A1, A2 = gpu.ActQ(wtype, n, 1), gpu.ActQ(wtype, n, 1)
    gpu.lib().b200_layernorm_q(xd.ptr, n, rad.ptr, rbd.ptr, gd[0].ptr, gd[1].ptr, A1.h, gd[2].ptr if dual else None, gd[3].ptr if dual else None,
                               A2.h if dual else None, n, 1)
    xs = (ra + rb) + x                                      # libfalcon.cpp:2399-2400: (ffn + attn) + inpL, fp32
    assert np.array_equal(xd.download(np.float32, (n,)), xs)
    at = po.VEC_DOT_TYPE[wtype]
    bb, blk = po.BLOCK_BYTES[at], po.BLOCK_ELEMS[at]
    for A, g, b in ((A1, g1, b1), (A2, g2, b2))[:2 if dual else 1]:
        q, d, s, bs = A.download()
        ref = orc.quantize_act(wtype, orc.layernorm(xs[None, :], g, b)).reshape(n // blk, bb)
        if at == po.Q8_K:                                   # {f32 d; int8 qs[256]; int16 bsums[16]}
            assert np.array_equal(d[0].view(np.uint32), ref[:, :4].copy().view(np.uint32)[:, 0])
            assert np.array_equal(q[0].reshape(-1, 256), ref[:, 4:260].view(np.int8))
            assert np.array_equal(bs[0].reshape(-1, 16), ref[:, 260:292].copy().view(np.int16))
        else:                                               # {f16 d; int8 qs[32]}
            assert np.array_equal(d[0], ref[:, :2].copy().view(np.float16)[:, 0].astype(np.float32))
            assert np.array_equal(q[0].reshape(-1, 32), ref[:, 2:34].view(np.int8))


def _attention_ref(orc, qkv, kc, vc, n_head, n_head_kv, n_past, n_ctx_rope):
    """numpy restatement of libfalcon.cpp:2229-2366 for the new tokens `qkv` over cache rows [0, n_past): returns (out, k_new, v_new)"""
    hd = 64
    n_tok = qkv.shape[0]
    q3 = qkv.reshape(n_tok, -1, hd)
    q = orc.rope_neox(q3[:, :n_head], n_past, n_ctx_rope)
    k = orc.rope_neox(q3[:, n_head:n_head + n_head_kv], n_past, n_ctx_rope)
    v = q3[:, n_head + n_head_kv:]
    K = np.concatenate([kc[:n_past], k]); V = np.concatenate([vc[:n_past], v])
    grp = n_head // n_head_kv
    out = np.zeros((n_tok, n_head, hd), np.float32)
    for kvh in range(n_head_kv):
        Kh, Vh = K[:, kvh], V[:, kvh]                         # [T][64]
        for h in range(kvh * grp, (kvh + 1) * grp):
            S = (q[:, h] @ Kh.T).astype(np.float32) * np.float32(0.125)         # [n_tok][T]
            for t in range(n_tok):
                S[t, n_past + t + 1:] = -np.inf               # ggml.c:12342-12348
            P = orc.soft_max(S)
            out[:, h] = P @ Vh
    return out, k, v


@pytest.mark.parametrize("n_head,n_head_kv,wtype", [(128, 8, po.Q4_K), (71, 1, po.Q4_0), (232, 8, po.Q4_K), (128, 8, po.Q4_0)])
@pytest.mark.parametrize("n_past", [0, 300, 2040, 8184])
def test_attention_decode_node(gpu, orc, n_head, n_head_kv, wtype, n_past):
    """the decode step's attention node at the real head geometry: G = 16 (Falcon-40B, Q8_K blocks folded into the combine step),
    G = 71 (Falcon-7B, 5 head groups, Q8_0 folded), G = 29 (Falcon-180B: two ragged groups, Q8_K not foldable -> own kernel).
    fp32 output within the decode bound of test_attention; the quantised hand-over to `wo` is BIT-EXACT with quantize_row_q8_* of the
    kernel's own fp32 output row (ggml.c:11462-11476)."""
    rng = np.random.default_rng(n_head + n_past)
    hd, n_ctx = 64, 8192
    QKV = (n_head + 2 * n_head_kv) * hd
    kc = np.zeros((n_ctx, n_head_kv, hd), np.float32)
    vc = np.zeros_like(kc)
    kc[:n_past] = rng.standard_normal((n_past, n_head_kv, hd)).astype(np.float32)
    vc[:n_past] = rng.standard_normal((n_past, n_head_kv, hd)).astype(np.float32)
    qkv = rng.standard_normal((1, QKV)).astype(np.float32)
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=kc), gpu.DevBuf(src=vc), gpu.DevBuf(n_head * hd * 4)
    A = gpu.ActQ(wtype, n_head * hd, 1)
    folded = gpu.lib().b200_attention_decode(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, hd, n_past, n_ctx, n_ctx, A.h)
    at = po.VEC_DOT_TYPE[wtype]
    assert folded == (1 if (at != po.Q8_K or (n_head // n_head_kv) % 4 == 0) else 0)
    got = od.download(np.float32, (1, n_head, hd))
    want, k_new, v_new = _attention_ref(orc, qkv, kc, vc, n_head, n_head_kv, n_past, n_ctx)
    assert np.allclose(kd.download(np.float32, kc.shape)[n_past], k_new[0], rtol=0, atol=1e-5 * max(1.0, np.abs(k_new).max()))
    assert np.array_equal(vd.download(np.float32, vc.shape)[n_past], v_new[0])
    assert np.allclose(got, want, rtol=0, atol=2e-3)
    assert np.median(np.abs(got - want)) < 2e-6
    q, d, s, bs = A.download()
    bb, blk = po.BLOCK_BYTES[at], po.BLOCK_ELEMS[at]
    ref = orc.quantize_act(wtype, got.reshape(1, -1)).reshape(-1, bb)
    if at == po.Q8_K:
        assert np.array_equal(d[0].view(np.uint32), ref[:, :4].copy().view(np.uint32)[:, 0])
        assert np.array_equal(q[0].reshape(-1, 256), ref[:, 4:260].view(np.int8))
        assert np.array_equal(bs[0].reshape(-1, 16), ref[:, 260:292].copy().view(np.int16))
    else:
        assert np.array_equal(d[0], ref[:, :2].copy().view(np.float16)[:, 0].astype(np.float32))
        assert np.array_equal(q[0].reshape(-1, 32), ref[:, 2:34].view(np.int8))


@pytest.mark.parametrize("n_head,n_head_kv,n_tok,n_past", [(128, 8, 512, 1536), (128, 8, 200, 700), (71, 1, 130, 1918), (232, 8, 64, 4032)])
def test_prompt_attention_many_key_tiles(gpu, orc, n_head, n_head_kv, n_tok, n_past):
    """wgmma prompt attention with up to 32 key tiles of 128 (BASELINE config 3 runs 512-token chunks up to T = 2048) against the
    numpy / oracle restatement.  Tolerance: Q, K, V are rounded to fp16 (2^-11 relative) -> atol 5e-3, median 5e-4 on O(1) outputs."""
    rng = np.random.default_rng(n_tok + n_past)
    hd, n_ctx = 64, n_past + n_tok
    QKV = (n_head + 2 * n_head_kv) * hd
    kc = np.zeros((n_ctx, n_head_kv, hd), np.float32)
    vc = np.zeros_like(kc)
    kc[:n_past] = rng.standard_normal((n_past, n_head_kv, hd)).astype(np.float32)
    vc[:n_past] = rng.standard_normal((n_past, n_head_kv, hd)).astype(np.float32)
    qkv = rng.standard_normal((n_tok, QKV)).astype(np.float32)
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=kc), gpu.DevBuf(src=vc), gpu.DevBuf(n_tok * n_head * hd * 4)
    gpu.lib().b200_attention(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, hd, n_tok, n_past, n_ctx, 2048)
    got = od.download(np.float32, (n_tok, n_head, hd))
    want, _, _ = _attention_ref(orc, qkv, kc, vc, n_head, n_head_kv, n_past, 2048)
    assert np.allclose(got, want, rtol=0, atol=5e-3), float(np.abs(got - want).max())
    assert np.median(np.abs(got - want)) < 5e-4


@pytest.mark.parametrize("t,K,M,N", [(po.Q4_K, 8192, 256, 512), (po.Q4_K, 32768, 128, 512), (po.Q4_0, 4544, 192, 300), (po.Q3_K, 8192, 128, 256)])
def test_full_k_gemm_against_oracle_columns(gpu, orc, t, K, M, N):
    """b200_mul_mat (N > 8: quantise -> fp16 -> wgmma GEMM with fused dequantisation) at the real contraction lengths against the
    ORACLE's mul_mat (not against our own CUDA-core kernel): |diff| <= 2e-3 * sum_k |w_k x_k| per output (fp16 rounding of both operands,
    2^-11 each, random signs) and a tight median."""
    rng = np.random.default_rng(K + M)
    wq = ggcc.random_blocks(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    W = gpu.Weight(t, K, M, wq)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(N * M * 4)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, N, yd.ptr, M)
    got = yd.download(np.float32, (N, M))
    want = orc.mul_mat(t, wq, K, M, x, nthreads=NTHREADS)
    mag = np.abs(x) @ np.abs(orc.dequantize(t, wq, K)).T
    assert np.all(np.abs(got - want) <= 2e-3 * mag), float((np.abs(got - want) / mag).max())
    assert np.median(np.abs(got - want) / mag) < 1e-4


def test_streaming_loader_at_real_widths(gpu, tmp_path):
    """b200_falcon_load_ggcc (mmap -> pinned ring -> cudaMemcpyAsync -> planar repack, six host threads) on a 0.8 GB file whose matrices
    span many 32 MB chunks: the loaded engine is bit-identical to one filled tensor by tensor"""
    hp = GEOM["40b"]
    tensors = random_model(hp, po.Q4_K, seed=MODEL_SEED["40b"] + po.Q4_K)
    path = str(tmp_path / "m40.ggcc")
    ggcc.write_ggcc(path, hp, tensors, ftype=15)
    a, b = gpu.Falcon(hp, n_ctx=64, n_batch=4), gpu.Falcon(hp, n_ctx=64, n_batch=4)
    a.load_ggcc(path)
    secs, nbytes = a.load_stats()
    assert nbytes == sum(ggcc.tensor_nbytes(t, ne) for n, (t, ne, _) in tensors.items() if len(ne) == 2) and secs > 0
    b.set_tensors(tensors)
    toks = np.array([11, 200, 300], np.int32)
    assert np.array_equal(a.eval(toks, 0, all_logits=True), b.eval(toks, 0, all_logits=True))
    assert np.array_equal(a.eval(toks[:1], 3), b.eval(toks[:1], 3))
    a.free(); b.free()


def test_release_cached_models():
    for k in list(_models):
        f, o = _models.pop(k)
        f.free()
