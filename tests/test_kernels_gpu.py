"""-m gpu parity tests of the kernel-level C ABI (include/ggml_b200.h part A) against the oracle.

Bars: bit-exact for integer/byte work (block dequantisation, activation codes + scales); mat-vec = exact integer
block dots, so only fp32 summation order differs from the CPU -> |err| <= 2e-5 * sum_k |w_k x_k| (stated per test);
float ops (LayerNorm, GELU, RoPE, softmax/attention) within the tolerances written next to each assert.
"""
import os
import numpy as np
import pytest
import pyoracle as po

pytestmark = pytest.mark.gpu

ALL_TYPES = po.WEIGHT_TYPES


def _weights(orc, t, M, K, seed, scale=0.05):
    rng = np.random.default_rng(seed)
    w = (scale * rng.standard_normal((M, K))).astype(np.float32)
    return orc.quantize(t, w)


@pytest.mark.parametrize("t", ALL_TYPES + [po.F16, po.F32])
def test_dequantize_bit_exact(gpu, orc, t):
    """device planar repack + dequant_elem == dequantize_row_q* bit for bit (ggml.c:1509-1619, k_quants.c:344-877)"""
    M, K = 37, 1024
    wq = _weights(orc, t, M, K, seed=t)
    W = gpu.Weight(t, K, M, wq)
    got = W.dequantize()
    want = orc.dequantize(t, wq, K)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    rows = np.array([5, 0, 36, 5], np.int32)      # ggml_get_rows with repeats
    assert np.array_equal(W.dequantize(rows).view(np.uint32), want[rows].view(np.uint32))


def test_dequantize_unaligned_rows(gpu, orc):
    """K = 4544 (Falcon-7B): Q4_0 rows are 2556 B, not a multiple of 16 -- the planar layout must still be exact"""
    M, K = 19, 4544
    wq = _weights(orc, po.Q4_0, M, K, seed=3)
    got = gpu.Weight(po.Q4_0, K, M, wq).dequantize()
    assert np.array_equal(got.view(np.uint32), orc.dequantize(po.Q4_0, wq, K).view(np.uint32))


@pytest.mark.parametrize("t", [po.Q4_0, po.Q4_1, po.Q4_K])
def test_activation_quantization_bit_exact(gpu, orc, t):
    """codes, scales and block sums == quantize_row_q8_0 (x86 body) / q8_1 / q8_K_reference"""
    N, K = 5, 2048
    rng = np.random.default_rng(11)
    x = rng.standard_normal((N, K)).astype(np.float32) * np.array([1, 10, 0.01, 100, 1], np.float32)[:, None]
    x[4, :256] = 0.0                      # an all-zero block
    x[4, 300], x[4, 301] = 5.0, -5.0      # +/- tie on the block maximum: first one wins
    for blk in (32, 256):                 # the pair is the maximum magnitude of its 32-block and of its 256-block
        b0 = 300 // blk * blk
        a = np.abs(x[4, b0:b0 + blk])
        assert list(np.flatnonzero(a == a.max()) + b0) == [300, 301]
    xd = gpu.DevBuf(src=x)
    A = gpu.ActQ(t, K, N)
    A.quantize(xd.ptr)
    q, d, s, bs = A.download()
    ref = orc.quantize_act(t, x)
    at = po.VEC_DOT_TYPE[t]
    bb, blk = po.BLOCK_BYTES[at], po.BLOCK_ELEMS[at]
    r = ref.reshape(N, K // blk, bb)
    if at == po.Q8_K:
        assert np.array_equal(d.view(np.uint32), r[:, :, 0:4].copy().view(np.uint32).reshape(N, -1))
        assert np.array_equal(q, r[:, :, 4:260].copy().view(np.int8).reshape(N, K))
        rbs = r[:, :, 260:292].copy().view(np.int16).reshape(N, -1)
        nz = np.repeat(d != 0, 16, axis=1)              # the reference leaves bsums of all-zero blocks unwritten
        assert np.array_equal(bs[nz], rbs[nz]) and np.all(bs[~nz] == 0)
    elif at == po.Q8_0:
        dref = r[:, :, 0:2].copy().view(np.float16).astype(np.float32).reshape(N, -1)
        assert np.array_equal(d, dref)
        assert np.array_equal(q, r[:, :, 2:34].copy().view(np.int8).reshape(N, K))
        assert np.array_equal(bs, q.reshape(N, -1, 32).astype(np.int32).sum(-1).astype(np.int16))
    else:
        assert np.array_equal(d.view(np.uint32), r[:, :, 0:4].copy().view(np.uint32).reshape(N, -1))
        assert np.array_equal(s.view(np.uint32), r[:, :, 4:8].copy().view(np.uint32).reshape(N, -1))
        assert np.array_equal(q, r[:, :, 8:40].copy().view(np.int8).reshape(N, K))


def _mmv_check(gpu, orc, t, M, K, N, seed, epi=0):
    rng = np.random.default_rng(seed)
    wq = _weights(orc, t, M, K, seed)
    x = rng.standard_normal((N, K)).astype(np.float32)
    W = gpu.Weight(t, K, M, wq)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(N * M * 4)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, N, yd.ptr, M)
    got = yd.download(np.float32, (N, M))
    want = orc.mul_mat(t, wq, K, M, x)
    # |sum_k w x| error budget: fp32 reassociation of K/32 (or K/256) exactly-computed block terms
    wd = np.abs(orc.dequantize(t, wq, K))
    budget = 2e-5 * (wd @ np.abs(x).T).T + 1e-6
    err = np.abs(got - want)
    assert np.all(err <= budget), (po.TYPE_NAMES[t], float(err.max()), float(budget[err.argmax() // M, err.argmax() % M]))
    return got, want


@pytest.mark.parametrize("t", ALL_TYPES)
def test_mat_vec_all_types(gpu, orc, t):
    _mmv_check(gpu, orc, t, M=301, K=2048, N=1, seed=100 + t)


@pytest.mark.parametrize("t,K,M", [(po.Q4_K, 8192, 1024), (po.Q4_0, 4544, 263), (po.Q3_K, 8192, 130), (po.Q6_K, 1024, 65), (po.Q4_K, 32768, 96)])
def test_mat_vec_model_shapes(gpu, orc, t, K, M):
    _mmv_check(gpu, orc, t, M=M, K=K, N=1, seed=7)


@pytest.mark.parametrize("t", [po.Q4_0, po.Q4_K, po.Q5_1])
def test_mat_vec_small_batch(gpu, orc, t):
    _mmv_check(gpu, orc, t, M=200, K=1024, N=5, seed=9)


@pytest.mark.parametrize("t", [po.F16, po.F32])
def test_mat_vec_float_weights(gpu, orc, t):
    rng = np.random.default_rng(5)
    M, K, N = 77, 1000 if t == po.F32 else 1024, 2
    w = (0.05 * rng.standard_normal((M, K))).astype(np.float32)
    wq = orc.quantize(t, w)
    x = rng.standard_normal((N, K)).astype(np.float32)
    W = gpu.Weight(t, K, M, wq)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(N * M * 4)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, N, yd.ptr, M)
    got = yd.download(np.float32, (N, M))
    want = orc.mul_mat(t, wq, K, M, x)
    assert np.allclose(got, want, rtol=0, atol=2e-5 * np.abs(w).sum(1).max())


def test_mat_vec_gelu_and_residual_epilogues(gpu, orc):
    t, M, K = po.Q4_K, 300, 1024
    rng = np.random.default_rng(21)
    wq = _weights(orc, t, M, K, 21, scale=0.2)
    x = rng.standard_normal((1, K)).astype(np.float32)
    r1, r2 = rng.standard_normal(M).astype(np.float32), rng.standard_normal(M).astype(np.float32)
    W = gpu.Weight(t, K, M, wq)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(M * 4)
    A = gpu.ActQ(t, K, 1)
    A.quantize(xd.ptr)
    base = orc.mul_mat(t, wq, K, M, x)[0]
    gpu.lib().b200_mul_mat_vec_q(W.h, A.h, yd.ptr, M, 1, None, None)
    got = yd.download(np.float32, (M,))
    want = orc.gelu(base)
    # GELU goes through fp16: allow one fp16 ulp where the fp32 dot differs in its last bits
    assert np.all(np.abs(got - want) <= np.maximum(np.abs(want) * 2.0 ** -10, 1e-7))
    assert np.mean(got == want) > 0.98
    r1d, r2d = gpu.DevBuf(src=r1), gpu.DevBuf(src=r2)
    gpu.lib().b200_mul_mat_vec_q(W.h, A.h, yd.ptr, M, 2, r1d.ptr, r2d.ptr)
    got = yd.download(np.float32, (M,))
    assert np.allclose(got, (base + r1) + r2, rtol=1e-6, atol=1e-5)


def test_layernorm(gpu, orc):
    """double-accumulated LayerNorm (ggml.c:10568-10595): bit-exact except where the parallel double sum rounds differently"""
    rng = np.random.default_rng(2)
    rows, n = 6, 8192
    x = (rng.standard_normal((rows, n)) * 3 + 0.5).astype(np.float32)
    g = (1 + 0.1 * rng.standard_normal(n)).astype(np.float32)
    b = (0.01 * rng.standard_normal(n)).astype(np.float32)
    xd, gd, bd, yd = gpu.DevBuf(src=x), gpu.DevBuf(src=g), gpu.DevBuf(src=b), gpu.DevBuf(rows * n * 4)
    gpu.lib().b200_layernorm(xd.ptr, n, gd.ptr, bd.ptr, yd.ptr, n, n, rows)
    got = yd.download(np.float32, (rows, n))
    want = orc.layernorm(x, g, b)
    assert np.allclose(got, want, rtol=0, atol=1e-6)           # tolerance: 1 ulp of O(1..8) values
    assert np.mean(got == want) > 0.99
    gpu.lib().b200_layernorm(xd.ptr, n, None, None, yd.ptr, n, n, rows)
    assert np.allclose(yd.download(np.float32, (rows, n)), orc.norm(x), rtol=0, atol=1e-6)


def test_gelu(gpu, orc):
    x = np.linspace(-12, 12, 100001).astype(np.float32)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(x.nbytes)
    gpu.lib().b200_gelu(xd.ptr, yd.ptr, x.size)
    got, want = yd.download(np.float32, x.shape), orc.gelu(x)
    # fp16-LUT semantics: equal except where device tanhf and glibc tanhf straddle an fp16 rounding boundary (1 fp16 ulp)
    assert np.all(np.abs(got - want) <= np.maximum(np.abs(want) * 2.0 ** -10, 6e-8))
    assert np.mean(got == want) > 0.999


@pytest.mark.parametrize("n_ctx_rope,n_past", [(64, 0), (2048, 1234), (8192, 8000)])
def test_rope_neox_ntk(gpu, orc, n_ctx_rope, n_past):
    rng = np.random.default_rng(4)
    n_tok, n_head, hd = 3, 9, 64
    x = rng.standard_normal((n_tok, n_head, hd)).astype(np.float32)
    xd = gpu.DevBuf(src=x)
    gpu.lib().b200_rope_neox(xd.ptr, n_tok, n_head, hd, n_head * hd, n_past, n_ctx_rope, 1, 2.0, 0)
    got = xd.download(np.float32, x.shape)
    want = orc.rope_neox(x, n_past, n_ctx_rope)
    # tolerance: device vs glibc cosf/sinf differ by <= 2 ulp on arguments up to n_past radians
    assert np.allclose(got, want, rtol=0, atol=3e-6 * np.abs(x).max())


@pytest.mark.parametrize("n_head,n_head_kv,n_tok,n_past", [(4, 2, 1, 0), (4, 2, 1, 37), (8, 1, 1, 200), (16, 8, 5, 11), (4, 2, 7, 0),
                                                           (32, 2, 40, 90), (71, 1, 3, 60), (16, 8, 100, 0)])
def test_attention(gpu, orc, n_head, n_head_kv, n_tok, n_past):
    """rope + KV append + causal GQA attention vs a numpy restatement built from the oracle's rope and softmax"""
    rng = np.random.default_rng(6)
    hd, n_ctx = 64, 256
    QKV = (n_head + 2 * n_head_kv) * hd
    kc = np.zeros((n_ctx, n_head_kv, hd), np.float32)   # decode (n_tok == 1) and prefill (n_tok > 1) kernels
    vc = np.zeros_like(kc)
    kc[:n_past] = rng.standard_normal((n_past, n_head_kv, hd)).astype(np.float32)
    vc[:n_past] = rng.standard_normal((n_past, n_head_kv, hd)).astype(np.float32)
    qkv = rng.standard_normal((n_tok, QKV)).astype(np.float32)
    qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=kc), gpu.DevBuf(src=vc), gpu.DevBuf(n_tok * n_head * hd * 4)
    os.environ["B200_ATTN_TC"] = "1"            # tensor-core kernel for every n_tok > 1 (the engine uses it for n_tok > 8)
    try:
        gpu.lib().b200_attention(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, hd, n_tok, n_past, n_ctx, n_ctx)
    finally:
        del os.environ["B200_ATTN_TC"]
    got = od.download(np.float32, (n_tok, n_head, hd))
    # oracle
    q3 = qkv.reshape(n_tok, -1, hd)
    q = orc.rope_neox(q3[:, :n_head], n_past, n_ctx)
    k = orc.rope_neox(q3[:, n_head:n_head + n_head_kv], n_past, n_ctx)
    kc[n_past:n_past + n_tok] = k
    vc[n_past:n_past + n_tok] = q3[:, n_head + n_head_kv:]
    assert np.allclose(kd.download(np.float32, kc.shape), kc, rtol=0, atol=1e-5)
    assert np.array_equal(vd.download(np.float32, vc.shape), vc)
    want = np.zeros_like(got)
    grp = n_head // n_head_kv
    for t in range(n_tok):
        T = n_past + t + 1
        for h in range(n_head):
            s = (kc[:T, h // grp] @ q[t, h]).astype(np.float32) * np.float32(0.125)
            p = orc.soft_max(s[None, :])[0]
            want[t, h] = p @ vc[:T, h // grp]
    # tolerance: the exp LUT rounds (s - max) to fp16, so a 1e-6 difference in a score can move one probability
    # by one fp16 ulp (2^-11 relative); outputs are O(1) averages of V
    if n_tok == 1:                      # decode kernel: fp32 throughout
        assert np.allclose(got, want, rtol=0, atol=2e-3)
        assert np.median(np.abs(got - want)) < 2e-6
    else:                               # tensor-core kernel: Q, K, V rounded to fp16 (2^-11 relative), fp32 accumulation, P exact
        assert np.allclose(got, want, rtol=0, atol=5e-3)
        assert np.median(np.abs(got - want)) < 5e-4
        os.environ["B200_ATTN_SIMT"] = "1"      # the CUDA-core fp32 kernels it replaces keep the tight bound
        qd2 = gpu.DevBuf(src=qkv)
        try:
            gpu.lib().b200_attention(qd2.ptr, kd.ptr, vd.ptr, od.ptr, n_head, n_head_kv, hd, n_tok, n_past, n_ctx, n_ctx)
        finally:
            del os.environ["B200_ATTN_SIMT"]
        got = od.download(np.float32, (n_tok, n_head, hd))
        assert np.allclose(got, want, rtol=0, atol=2e-3)
        assert np.median(np.abs(got - want)) < 2e-6


@pytest.mark.parametrize("t,M,K,N,gelu", [(po.Q4_K, 256, 512, 40, 0), (po.Q4_K, 1000, 1024, 300, 0), (po.Q4_K, 384, 2048, 512, 1),
                                          (po.Q4_0, 200, 256, 17, 0), (po.Q6_K, 128, 512, 64, 0), (po.Q4_K, 128, 8192, 9, 0), (po.Q4_K, 640, 1024, 512, 0),
                                          (po.Q6_K, 300, 512, 260, 0), (po.Q4_K, 520, 2048, 400, 1),       # N > 256: two token tiles
                                          (po.Q4_0, 300, 4544, 512, 0), (po.Q3_K, 520, 2048, 400, 0), (po.Q3_K, 130, 1024, 77, 1), (po.Q4_0, 71, 576, 130, 0)])
def test_tensor_core_gemm_matches_cuda_core_gemm(gpu, orc, t, M, K, N, gelu):
    """wgmma kernel vs the CUDA-core kernel on identical fp16 operands: only the fp32 accumulation order differs.
    Then both against the exact fp64 product of the fp16-rounded operands."""
    rng = np.random.default_rng(M + K + N)
    wq = _weights(orc, t, M, K, seed=3)
    xh = rng.standard_normal((N, K)).astype(np.float16)
    W = gpu.Weight(t, K, M, wq)
    xd, y0, y1 = gpu.DevBuf(src=xh), gpu.DevBuf(N * M * 4), gpu.DevBuf(N * M * 4)
    y1.zero()
    assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, y0.ptr, M, gelu, 0) == 1
    assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, y1.ptr, M, gelu, 1) == 1
    a, b = y0.download(np.float32, (N, M)), y1.download(np.float32, (N, M))
    wd = orc.dequantize(t, wq, K).astype(np.float16).astype(np.float64)
    exact = xh.astype(np.float64) @ wd.T
    budget = 3e-6 * (np.abs(xh.astype(np.float64)) @ np.abs(wd).T) + 1e-6
    if gelu:
        exact = orc.gelu(exact.astype(np.float32)).astype(np.float64)
        budget = np.maximum(budget, np.abs(exact) * 2.0 ** -9 + 1e-6)        # fp16 rounding of the GELU input and of its output
    assert np.all(np.abs(b - exact) <= budget), float(np.abs(b - exact).max())
    assert np.all(np.abs(a - exact) <= budget), float(np.abs(a - exact).max())


@pytest.mark.parametrize("t,K,M", [(po.Q4_K, 8192, 32768), (po.Q4_K, 512, 768), (po.Q4_0, 4544, 18176)])
def test_matvec_chain_quantises_output_for_next_matmul(gpu, orc, t, K, M):
    """ffn_up -> ffn_down hand-over: the mat-vec's own CTAs quantise the (GELU'd) output row, 256 values at a time, as
    they finish.  Codes / scales / sums must equal the standalone quantiser run on the same fp32 row, bit for bit,
    launch after launch (the chunk counters re-arm themselves)."""
    rng = np.random.default_rng(K + M)
    wq = _weights(orc, t, M, K, seed=9)
    W = gpu.Weight(t, K, M, wq)
    A_in, A_out, A_ref = gpu.ActQ(t, K, 1), gpu.ActQ(t, M, 1), gpu.ActQ(t, M, 1)
    yd = gpu.DevBuf(M * 4)
    for it in range(3):
        x = rng.standard_normal(K).astype(np.float32)
        xd = gpu.DevBuf(src=x)
        A_in.quantize(xd.ptr)
        assert gpu.lib().b200_mul_mat_vec_q_chain(W.h, A_in.h, yd.ptr, 1, A_out.h) == 1
        y = yd.download(np.float32, (M,))
        gpu.lib().b200_mul_mat_vec_q(W.h, A_in.h, yd.ptr, M, 1, None, None)          # same kernel without the hand-over
        assert np.array_equal(y, yd.download(np.float32, (M,)))
        A_ref.quantize(yd.ptr)
        (q, d, _, bs), (q0, d0, _, bs0) = A_out.download(), A_ref.download()      # (the s plane exists for Q8_1 only)
        assert np.array_equal(q, q0) and np.array_equal(d, d0) and np.array_equal(bs, bs0)


@pytest.mark.parametrize("t,K,M", [(po.Q4_K, 8192, 65024), (po.Q4_K, 32768, 8192), (po.Q4_K, 8192, 32768), (po.Q4_0, 4544, 65024),
                                   (po.Q4_0, 18176, 4544), (po.Q3_K, 8192, 9216)])
def test_full_size_matvec_all_rows(gpu, orc, t, K, M):
    """BASELINE's real matrix shapes (Falcon-40B / 7B qkv, ffn, lm_head), every output row against the oracle's
    mul_mat_q_f32 restatement.  Weights are well-formed random blocks (any byte pattern is a valid block), so the integer
    block dots are exact on both sides and only the fp32 summation order differs."""
    import ggllm_cpp_b200.ggcc as ggcc
    rng = np.random.default_rng(K ^ M)
    wq = ggcc.random_blocks(t, M, K, rng)
    x = rng.standard_normal((1, K)).astype(np.float32)
    W = gpu.Weight(t, K, M, wq)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(M * 4)
    A = gpu.ActQ(t, K, 1); A.quantize(xd.ptr)
    gpu.lib().b200_mul_mat_vec_q(W.h, A.h, yd.ptr, M, 0, None, None)
    got = yd.download(np.float32, (M,))
    want = orc.mul_mat(t, wq, K, M, x)[0]
    scale = float(np.abs(want).max())
    assert np.isfinite(got).all() and scale > 0
    assert np.abs(got - want).max() <= 2e-5 * scale, (float(np.abs(got - want).max()), scale)
    assert np.median(np.abs(got - want)) <= 1e-6 * scale


@pytest.mark.parametrize("K,M,N", [(8192, 32768, 512), (32768, 8192, 512), (8192, 9216, 384)])
def test_full_size_gemm_tensor_core_vs_cuda_core(gpu, K, M, N):
    """BASELINE config 3 shapes (Falcon-40B ffn_up / ffn_down / qkv at n_batch 512): the wgmma kernel and the CUDA-core
    reference kernel read the same Q4_K blocks and the same fp16 activations; only the fp32 accumulation order differs."""
    import ggllm_cpp_b200.ggcc as ggcc
    rng = np.random.default_rng(K + M + N)
    wq = ggcc.random_blocks(po.Q4_K, M, K, rng)
    xh = rng.standard_normal((N, K)).astype(np.float16)
    W = gpu.Weight(po.Q4_K, K, M, wq)
    xd, y0, y1 = gpu.DevBuf(src=xh), gpu.DevBuf(N * M * 4), gpu.DevBuf(N * M * 4)
    y1.zero()
    assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, y0.ptr, M, 0, 0) == 1
    assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, y1.ptr, M, 0, 1) == 1
    a, b = y0.download(np.float32, (N, M)), y1.download(np.float32, (N, M))
    scale = float(np.abs(a).max())
    assert np.isfinite(b).all() and scale > 0
    # fp32 reassociation over K products (and the two-way K split of the wgmma kernel): grows like sqrt(K)
    grow = (K / 8192.0) ** 0.5
    assert np.abs(a - b).max() <= 1e-4 * grow * scale, (float(np.abs(a - b).max()), scale)
    assert np.median(np.abs(a - b)) <= 5e-6 * grow * scale, (float(np.median(np.abs(a - b))), scale)


@pytest.mark.parametrize("t", [po.Q4_0, po.Q4_K, po.Q2_K, po.Q3_K, po.Q5_K, po.Q6_K])
def test_device_weight_quantiser_bit_exact(gpu, orc, t):
    """b200_quantize_weights writes the reference quantiser's blocks bit for bit (ggml.c:927-962, k_quants.c:275-342, 396-470, 542-605,
    652-732, 781-843):
    normal, tiny, huge, zero, constant, one-sided and the reference test's 0.1 + 2 cos(i) data (tests/test-quantize-fns.cpp:26-32)"""
    K, rng = 4096, np.random.default_rng(t)
    rows = [rng.standard_normal(K), 1e-8 * rng.standard_normal(K), 1e8 * rng.standard_normal(K), np.zeros(K), np.full(K, 0.37),
            np.abs(rng.standard_normal(K)), -np.abs(rng.standard_normal(K)), 0.1 + 2.0 * np.cos(np.arange(K)),
            0.02 * rng.standard_normal(K), rng.standard_normal(K) * (rng.random(K) < 0.05)]
    w = np.stack(rows).astype(np.float32)
    want = orc.quantize(t, w)
    xd, out = gpu.DevBuf(src=w), gpu.DevBuf(want.nbytes)
    assert gpu.lib().b200_quantize_weights(t, xd.ptr, out.ptr, w.size) == 1
    got = out.download(np.uint8, want.shape)
    assert np.array_equal(got, want), int((got != want).sum())
    assert gpu.lib().b200_quantize_weights(po.Q8_0, xd.ptr, out.ptr, w.size) == 0       # no device quantiser for this type: the caller quantises on the host
