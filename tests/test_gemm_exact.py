"""CPU tests of the prompt GEMM's grid operands and numpy model (tests/gemm_exact.py) that the GPU tests compare against bit for bit.

  * the grid weights dequantise, through the oracle, to multiples of G that are exact in fp16, with the scale fields and sub-scales
    the builder meant, and codes over their whole range; the dispatcher's activation rows quantise to themselves
  * every case of the GPU parametrisation stays inside the headroom that makes fp32 accumulation exact in any order
  * every fault a producer or the K split typically has changes some output of every case it applies to
  * through b200_gemm_launch_shape, the parametrisation reaches every launch shape, and the edges of the tiling and the K split
"""
import os
import numpy as np
import pytest
import pyoracle as po
import mmv_exact as mx
import gemm_exact as gx


@pytest.fixture(scope="module", autouse=True)
def _lib():
    import ggllm_cpp_b200.binding as b
    if not os.path.exists(b.LIB_PATH):
        b.build()


def _sub_of_element(t, K):
    """the sub-block (scale index) of every element of a block"""
    n = 8 if t in (po.Q4_K, po.Q5_K) else 16
    return np.arange(mx.BE[t]) // (mx.BE[t] // n)


CODES = {po.Q4_0: (-8, 7), po.Q4_1: (0, 15), po.Q5_0: (-16, 15), po.Q5_1: (0, 31), po.Q8_0: (-128, 127), po.Q2_K: (0, 3),
         po.Q3_K: (-4, 3), po.Q4_K: (0, 15), po.Q5_K: (0, 31), po.Q6_K: (-32, 31)}


@pytest.mark.parametrize("t", gx.GRID_TYPES, ids=lambda t: po.TYPE_NAMES[t])
def test_grid_weights_dequantise_exactly(orc, t):
    M, K = 6, 2048
    wq = gx.grid_weights(t, M, K, np.random.default_rng(t))
    w = gx.dequant(t, wq, K)
    k = w / gx.G
    assert np.array_equal(k, np.round(k)) and np.abs(k).max() < 2048                # multiples of G, exact in fp16
    assert np.array_equal(w, w.astype(np.float16).astype(np.float64))
    if t == po.F16:
        return
    nb = K // mx.BE[t]
    d = mx._f16_field(wq, t, mx.D_OFF[t])
    want_d = gx.G * 2.0 ** ((np.arange(M)[:, None] + np.arange(nb)[None, :]) % 2)
    assert np.array_equal(d, want_d)
    assert np.all(d[:, 1:] != d[:, :-1]) and np.all(d[1:] != d[:-1])                 # neighbouring blocks and rows differ
    # the same blocks with d = 1 and min = 0: codes times sub-block scales, exact in the fp32 dequantiser
    bA = mx._set_f16(wq, t, mx.D_OFF[t], 1.0)
    if t in mx.M_OFF:
        bA = mx._set_f16(bA, t, mx.M_OFF[t], 0.0)
    A = orc.dequantize(t, bA, K).astype(np.float64).reshape(M, nb, mx.BE[t])
    B = np.zeros_like(A)
    if t in mx.M_OFF:
        dm = mx._f16_field(wq, t, mx.M_OFF[t])
        B = orc.dequantize(t, mx._set_f16(mx._set_f16(wq, t, mx.D_OFF[t], 0.0), t, mx.M_OFF[t], 1.0), K).astype(np.float64)
        B = B.reshape(M, nb, mx.BE[t])
        assert np.all(dm[:, 1:] != dm[:, :-1]) and np.all(dm[1:] != dm[:-1])
        assert np.array_equal(w.reshape(M, nb, -1), d[..., None] * A + dm[..., None] * B)
    else:
        assert np.array_equal(w.reshape(M, nb, -1), d[..., None] * A)
    sc, mins = gx.sub_scales(t, M, nb)
    if sc is None:
        codes = A
    else:
        s = sc.astype(np.float64)[:, :, _sub_of_element(t, K)]
        codes = A / s
        assert np.all(np.diff(sc.astype(np.int64), axis=-1) != 0)                      # neighbouring sub-blocks differ
        if mins is not None:                                                            # the min part is -min * sub-block min
            assert np.array_equal(B, -mins.astype(np.float64)[:, :, _sub_of_element(t, K)])
    assert np.array_equal(codes, np.round(codes))
    lo, hi = CODES[t]
    assert codes.min() == lo and codes.max() == hi                                      # the whole code range


@pytest.mark.parametrize("c", gx.MUL_MAT, ids=gx.case_id)
def test_dispatcher_activations_quantise_to_themselves(orc, c):
    """b200_mul_mat quantises its fp32 rows first: on grid_acts_q8 rows the codes times the scales are the rows themselves"""
    t, K, M, N = c
    x = gx.grid_acts_q8(t, 4, K, np.random.default_rng(K))
    q, d, _, _ = mx.act_from_blocks(t, orc.quantize_act(t, x), K)
    xd = q.astype(np.float64) * np.repeat(d.astype(np.float64), K // d.shape[1], axis=1)
    assert np.array_equal(xd, x.astype(np.float64))
    assert np.array_equal(xd.astype(np.float16).astype(np.float64), xd)


def _case(c, q8=False):
    t, K, M, N = c
    rng = np.random.default_rng(gx.case_seed(c))
    wq = gx.grid_weights(t, M, K, rng)
    x = gx.grid_acts_q8(t, N, K, rng) if q8 else gx.grid_acts(N, K, rng)
    return wq, x


ALL = [(c, False) for c in gx.TC + gx.GELU] + [(c, True) for c in gx.MUL_MAT]


@pytest.mark.parametrize("c,q8", ALL, ids=[gx.case_id(c) + ("-mul_mat" if q8 else "") for c, q8 in ALL])
def test_every_case_within_headroom(c, q8):
    """sum_k |w x| <= HEADROOM G for every output of every case (the largest M is checked on a sample of rows)"""
    t, K, M, N = c
    wq, x = _case(c, q8)
    rows = np.arange(M) if M <= 1024 else np.r_[0:256, M - 256:M]
    _, mag = gx.gemm_model(t, wq, K, x, rows=rows, mag=True)
    assert mag.max() <= gx.HEADROOM * gx.G, (mag.max() / gx.G)


@pytest.mark.parametrize("c", gx.TC, ids=gx.case_id)
def test_every_fault_is_visible(c):
    """for every fault that applies to the case's type and launch, the faulty model differs from the true Y in some output"""
    t, K, M, N = c
    wq, x = _case(c)
    (shape, _), = gx.launches(c)
    ks = shape[1] if shape else 1
    rows, toks = np.unique([0, 1, 2, M - 2, M - 1]), np.unique([0, 1, N - 1])
    y = gx.gemm_model(t, wq, K, x, ks, rows=rows, toks=toks)
    silent = [f for f in gx.faults_for(t, ks, K) if np.array_equal(gx.gemm_model(t, wq, K, x, ks, fault=f, rows=rows, toks=toks), y)]
    assert not silent, silent


def _reached():
    """(producer, BN, ksplit) and the K-block facts of every wgmma call the GPU parametrisation makes; and whether the CUDA-core
    fallback runs"""
    shapes, facts, simt = set(), dict(KB=set(), uneven=False, q3_mid=False, q4_mid=False, m_tail=set(), n_ragged=False), False
    for cases, gelu in ((gx.TC, False), (gx.GELU, True), (gx.MUL_MAT, False)):
        for c in cases:
            t, K, M, N = c
            for s, n in gx.launches(c, gelu):
                if s is None:
                    simt = True
                    continue
                bn, ks, prod = s
                shapes.add((prod, bn, ks))
                hv = gx.halves(K, ks)
                facts["KB"] |= {kb for _, kb in hv}
                facts["uneven"] |= ks == 2 and hv[0][1] != hv[1][1]
                facts["q3_mid"] |= t == po.Q3_K and ks == 2 and hv[1][0] % 4 == 2
                facts["q4_mid"] |= t == po.Q4_K and ks == 2 and hv[1][0] % 4 == 2
                r = M % gx.BM
                facts["m_tail"].add("full" if r == 0 else "one" if r == 1 else "<=64" if r <= 64 else ">64")
                facts["n_ragged"] |= n % bn != 0
    return shapes, facts, simt


def test_parametrisation_reaches_every_launch_shape():
    """every (producer, BN, ksplit) launch_gemm_tc can choose, and the CUDA-core fallback; K blocks per CTA 1, 2, 3, ST and ST + 1;
    an uneven split; Q3_K and Q4_K halves starting at kb0 = 2 (mod 4); an empty, partial and full second consumer warpgroup; N % BN"""
    possible = set()
    for t in (po.Q4_K, po.Q4_0, po.Q3_K, po.Q6_K):
        for K in (256, 512, 8192):
            for M in (1, 129, 20000):
                for N in (9, 64, 65, 128, 129, 512):
                    for gelu in (False, True):
                        s = gx.launches((t, K, M, N), gelu)[0][0]
                        possible.add((s[2], s[0], s[1]))
    assert len(possible) == 24, sorted(possible)
    assert gx.launches((po.Q4_0, 4576, 10, 100))[0][0] is None
    import ggllm_cpp_b200.binding as b
    assert b.gemm_launch_shape(po.Q4_0, 4544, 10, 100, 4548) is None and b.gemm_launch_shape(po.Q4_0, 4544, 10, 513) is None
    shapes, facts, simt = _reached()
    assert not possible - shapes, sorted(possible - shapes)
    assert simt
    assert {1, 2, 3, gx.ST, gx.ST + 1} <= facts["KB"], facts["KB"]
    assert facts["uneven"] and facts["q3_mid"] and facts["q4_mid"] and facts["n_ragged"]
    assert {"one", "<=64", ">64"} <= facts["m_tail"], facts["m_tail"]
    assert any(c[1] in (8192, 14848, 32768) and gx.launches(c)[0][0][1] == 2 for c in gx.TC)
    assert any(c[1] in (8192, 14848, 32768) and gx.launches(c, g)[0][0][1] == 1 for cs, g in ((gx.TC, False), (gx.GELU, True)) for c in cs)
    assert {n for c in gx.MUL_MAT for n in [c[3]]} >= {513, 1000, 1025}
