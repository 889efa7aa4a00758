"""-m gpu: every launch shape of the decode mat-vec, per output, against the exact restatement of tests/mmv_exact.py; and row strides
on every mat-mul entry point.

The restatement reads the quantised activation back from the device (its codes and scales are first checked bit for bit against
the oracle's quantiser), computes each piece's integer dot exactly, and bounds the kernel's fp32 error by the roundings of one piece
term plus the longest addition chain of the shape that b200_mmv_launch_shape reports.  Every output must lie within that bound.
The largest error / bound ratio per kernel family and shape is printed at the end of the module (pytest -s).
"""
import collections
import os
import numpy as np
import pytest
import pyoracle as po
import mmv_exact as mx

gpu_mark = pytest.mark.gpu
L4K, L40, L3K = po.Q4_K, po.Q4_0, po.Q3_K
RATIOS = collections.defaultdict(float)

# (type, K, M, N, environment switch): one K inside each branch of the launch-shape choice and one on each edge
FAST = [(L4K, 2048, 301, 1, None), (L4K, 8192, 9216, 1, None), (L4K, 4352, 37, 2, None), (L4K, 14848, 5, 8, None),
        (L4K, 16384, 37, 1, None), (L4K, 18432, 64, 2, None), (L4K, 32768, 8192, 1, None), (L4K, 59392, 37, 1, None),
        (L4K, 65536, 5, 2, None), (L4K, 65792, 37, 1, None),
        (L40, 2048, 1, 1, None), (L40, 8192, 37, 8, None), (L40, 4544, 4672, 1, None), (L40, 14848, 37, 2, None),
        (L40, 16384, 5, 1, None), (L40, 18176, 4544, 1, None), (L40, 32768, 37, 1, None), (L40, 59392, 37, 2, None),
        (L40, 65536, 37, 1, None), (L40, 65568, 5, 1, None),
        (L3K, 8192, 9216, 1, None), (L3K, 14848, 37, 2, None), (L3K, 32768, 37, 8, None), (L3K, 59392, 37, 1, None),
        (L3K, 65792, 5, 1, None)]
# the generic ring kernel (mmv.cu): K with one, two and more work units per row and a ragged last unit, for every type; the
# types the tuned kernel covers go there through B200_MMV_GENERIC
GENERIC = [(t, K, 37, 2 if K == 8192 else 1, "B200_MMV_GENERIC" if t in (L4K, L40, L3K) else None)
           for t in po.WEIGHT_TYPES for K in ((4608, 8192, 18432, 32768) if mx.BE[t] == 256 else (4544, 8192, 18176, 32768))]
GENERIC += [(po.Q6_K, 8192, 9216, 1, None), (po.Q5_K, 32768, 8192, 1, None), (po.Q5_0, 4544, 4672, 1, None),
            (po.Q8_0, 18176, 4544, 1, None)]


def _shape(t, K, env):
    import ggllm_cpp_b200.binding as b
    return None if env == "B200_MMV_GENERIC" else b.mmv_launch_shape(t, K)


def _kernel(shape):
    return ("generic",) if shape is None else ("fast", shape[0], shape[1])


def _family(t, shape):
    return "%s %s" % (po.TYPE_NAMES[t], "generic" if shape is None else "fast NT%d J%d D%d" % shape)


class _env:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if self.name:
            os.environ[self.name] = "1"

    def __exit__(self, *a):
        if self.name:
            os.environ.pop(self.name, None)


def _setup(gpu, orc, t, K, M, N, seed):
    rng = np.random.default_rng(seed)
    wq = mx.swept_weights(t, M, K, rng)
    x = mx.swept_acts(t, N, K, rng)
    W = gpu.Weight(t, K, M, wq)
    xd = gpu.DevBuf(src=x)
    A = gpu.ActQ(t, K, N)
    A.quantize(xd.ptr)
    q, d, s, bs = A.download()
    rq, rd, rs, rbs = mx.act_from_blocks(t, orc.quantize_act(t, x), K)
    assert np.array_equal(q, rq) and np.array_equal(d.view(np.uint32), rd.view(np.uint32))
    if po.VEC_DOT_TYPE[t] == po.Q8_1:                       # the Q4_1 / Q5_1 dots read the sums s, not bs
        assert np.array_equal(s.view(np.uint32), rs.view(np.uint32))
    else:                                                   # the CPU leaves the bsums of an all-zero Q8_K block unwritten
        nz = np.repeat(d != 0, bs.shape[1] // d.shape[1], axis=1)
        assert np.array_equal(bs[nz], rbs[nz])
    return wq, x, W, A, (q, d, s)


def _check(t, K, wq, got, act, shape, epi=0, r=None):
    q, d, s = act
    fam = _family(t, shape)
    for n in range(got.shape[0]):
        y, bound, _, _ = mx.reference(t, wq, K, q[n], d[n], s[n], _kernel(shape))
        if epi == 1:
            ok = mx.gelu_ok(got[n], y, bound)
            assert ok.all(), (fam, n, int((~ok).sum()))
            continue
        if epi == 2:
            bound = mx.add2_bound(y, bound, r[0][n], r[1][n])
            y = y + r[0][n].astype(np.float64) + r[1][n].astype(np.float64)
        ratio = np.abs(got[n].astype(np.float64) - y) / bound
        RATIOS[fam + ("" if epi == 0 else " ADD2")] = max(RATIOS[fam + ("" if epi == 0 else " ADD2")], float(ratio.max()))
        assert np.all(ratio <= 1.0), (fam, n, float(ratio.max()), int(ratio.argmax()))


def _cid(c):
    return "%s-K%d-M%d-N%d%s" % (po.TYPE_NAMES[c[0]], c[1], c[2], c[3], "-" + c[4] if c[4] else "")


@gpu_mark
@pytest.mark.parametrize("case", FAST + GENERIC, ids=_cid)
def test_mat_vec_within_exact_bound(gpu, orc, case):
    t, K, M, N, env = case
    shape = _shape(t, K, env)
    wq, x, W, A, act = _setup(gpu, orc, t, K, M, N, seed=K + M + N)
    yd = gpu.DevBuf(N * M * 4)
    with _env(env):
        gpu.lib().b200_mul_mat_vec_q(W.h, A.h, yd.ptr, M, 0, None, None)
    _check(t, K, wq, yd.download(np.float32, (N, M)), act, shape)


EPI = [(L4K, 8192, 301, None), (L40, 14848, 301, None), (po.Q5_K, 18432, 301, None), (L40, 18176, 301, "B200_MMV_GENERIC")]


@gpu_mark
@pytest.mark.parametrize("epi", [1, 2], ids=["gelu", "add2"])
@pytest.mark.parametrize("case", EPI, ids=lambda c: "%s-K%d%s" % (po.TYPE_NAMES[c[0]], c[1], "-generic" if c[3] else ""))
def test_mat_vec_epilogues_within_exact_bound(gpu, orc, case, epi):
    t, K, M, env = case
    shape = _shape(t, K, env)
    wq, x, W, A, act = _setup(gpu, orc, t, K, M, 1, seed=K + epi)
    rng = np.random.default_rng(epi)
    r1, r2 = (rng.standard_normal((1, M)) * 64).astype(np.float32), (rng.standard_normal((1, M)) * 64).astype(np.float32)
    r1d, r2d, yd = gpu.DevBuf(src=r1), gpu.DevBuf(src=r2), gpu.DevBuf(M * 4)
    with _env(env):
        gpu.lib().b200_mul_mat_vec_q(W.h, A.h, yd.ptr, M, epi, r1d.ptr, r2d.ptr)
    _check(t, K, wq, yd.download(np.float32, (1, M)), act, shape, epi, (r1, r2))


@gpu_mark
def test_chain_at_falcon_180b_width(gpu, orc):
    """b200_mul_mat_vec_q_chain at Falcon-180B's ffn_up shape (K = 14848, M = 59392): the output row within the bound (its
    quantised hand-over is checked bit for bit against quantize_act in test_kernels_gpu.py)"""
    t, K, M = L4K, 14848, 59392
    wq, x, W, A, act = _setup(gpu, orc, t, K, M, 1, seed=180)
    A_out, yd = gpu.ActQ(t, M, 1), gpu.DevBuf(M * 4)
    assert gpu.lib().b200_mul_mat_vec_q_chain(W.h, A.h, yd.ptr, 0, A_out.h) == 1
    _check(t, K, wq, yd.download(np.float32, (1, M)), act, _shape(t, K, None))


@gpu_mark
@pytest.mark.parametrize("t,K,M", [(po.F16, 8192, 65024), (po.F16, 4544, 37), (po.F32, 8192, 8192), (po.F32, 4544, 37)])
def test_float_weight_mat_vec_within_exact_bound(gpu, orc, t, K, M):
    rng = np.random.default_rng(K + M)
    w = (0.02 * rng.standard_normal((M, K))).astype(np.float16 if t == po.F16 else np.float32)
    x = mx.swept_acts(po.Q4_0, 2, K, rng)
    W, xd, yd = gpu.Weight(t, K, M, w), gpu.DevBuf(src=x), gpu.DevBuf(2 * M * 4)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, 2, yd.ptr, M)
    got = yd.download(np.float32, (2, M))
    for n in range(2):
        y, bound = mx.f_reference(t, w, x[n])
        ratio = np.abs(got[n] - y) / bound
        RATIOS["%s mmv_f" % po.TYPE_NAMES[t]] = max(RATIOS["%s mmv_f" % po.TYPE_NAMES[t]], float(ratio.max()))
        assert np.all(ratio <= 1.0), (float(ratio.max()), int(ratio.argmax()))


def test_parametrisation_reaches_every_launch_shape():
    """every (NT, J, D) the launch-shape choice can return for Q4_K, Q4_0 and Q3_K is run by test_mat_vec_within_exact_bound;
    and K past 64 Ki goes to the generic kernel"""
    import ggllm_cpp_b200.binding as b
    if not os.path.exists(b.LIB_PATH):
        b.build()
    possible = set()
    for t in (L4K, L40, L3K):
        for K in range(256, 70000, 256):
            s = _shape(t, K, None)
            if s is not None:
                possible.add((t, s))
        assert _shape(t, 65536 + 256, None) is None
    reached = {(c[0], _shape(c[0], c[1], c[4])) for c in FAST}
    missing = possible - reached
    assert not missing, sorted(missing)
    assert len(possible) >= 15


# ---------------------------------------------------------------------------------------------------- row strides
NAN_BITS = np.uint32(0x7FC0DEAD)


def _strided_out(gpu, N, M, ys):
    buf = np.full((N, ys), NAN_BITS, np.uint32)
    return gpu.DevBuf(src=buf)


def _check_strided(got, want, M):
    """got [N][M + 8] uint32 bits, want [N][M] float32: outputs bit-identical, the 8 gap columns still hold the sentinel"""
    assert np.array_equal(got[:, :M], want.view(np.uint32)), int((got[:, :M] != want.view(np.uint32)).sum())
    assert np.all(got[:, M:] == NAN_BITS), int((got[:, M:] != NAN_BITS).sum())


@gpu_mark
@pytest.mark.parametrize("t,K,M,N", [(L4K, 2048, 300, 5), (L4K, 1024, 256, 40), (po.Q5_K, 4608, 77, 3), (po.Q6_K, 1024, 300, 130),
                                     (po.F16, 1024, 77, 2), (po.F32, 1000, 77, 3)])
def test_mul_mat_row_strides(gpu, orc, t, K, M, N):
    """b200_mul_mat with x_stride = K + 64 and y_stride = M + 8 (N <= 8: mat-vec; N > 8: the GEMM, which at M = 256, N = 40 splits
    K in two and clears Y first): same bits as the unstrided call, and the caller's gap columns untouched"""
    rng = np.random.default_rng(K + N)
    wq = (0.02 * rng.standard_normal((M, K))).astype(np.float16 if t == po.F16 else np.float32) if t in (po.F16, po.F32) \
        else mx.swept_weights(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    xs = np.full((N, K + 64), np.nan, np.float32)
    xs[:, :K] = x
    W = gpu.Weight(t, K, M, wq)
    xd, xsd, yd = gpu.DevBuf(src=x), gpu.DevBuf(src=xs), gpu.DevBuf(N * M * 4)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, N, yd.ptr, M)
    want = yd.download(np.float32, (N, M))
    assert np.isfinite(want).all()
    ysd = _strided_out(gpu, N, M, M + 8)
    gpu.lib().b200_mul_mat(W.h, xsd.ptr, K + 64, N, ysd.ptr, M + 8)
    _check_strided(ysd.download(np.uint32, (N, M + 8)), want, M)


@gpu_mark
@pytest.mark.parametrize("t,K,M,N,env", [(L4K, 14848, 300, 2, None), (L40, 4544, 77, 3, None), (po.Q5_0, 4544, 77, 2, None),
                                         (L3K, 8192, 300, 1, "B200_MMV_GENERIC")])
def test_mul_mat_vec_q_row_strides(gpu, orc, t, K, M, N, env):
    """b200_quantize_act from rows K + 64 apart and b200_mul_mat_vec_q into rows M + 8 apart"""
    rng = np.random.default_rng(K + M)
    wq = mx.swept_weights(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    xs = np.full((N, K + 64), np.nan, np.float32)
    xs[:, :K] = x
    W = gpu.Weight(t, K, M, wq)
    xd, xsd, yd = gpu.DevBuf(src=x), gpu.DevBuf(src=xs), gpu.DevBuf(N * M * 4)
    A, As = gpu.ActQ(t, K, N), gpu.ActQ(t, K, N)
    A.quantize(xd.ptr)
    As.quantize(xsd.ptr, K + 64)
    with _env(env):
        gpu.lib().b200_mul_mat_vec_q(W.h, A.h, yd.ptr, M, 0, None, None)
        want = yd.download(np.float32, (N, M))
        ysd = _strided_out(gpu, N, M, M + 8)
        gpu.lib().b200_mul_mat_vec_q(W.h, As.h, ysd.ptr, M + 8, 0, None, None)
    _check_strided(ysd.download(np.uint32, (N, M + 8)), want, M)


@gpu_mark
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("t,K,M,N", [(L4K, 1024, 256, 40), (L40, 4544, 300, 130), (po.Q6_K, 512, 300, 260)])
def test_mul_mat_f16_row_strides(gpu, orc, t, K, M, N, impl):
    """b200_mul_mat_f16 (impl 0 CUDA-core, impl 1 wgmma; M = 256, N = 40 takes the two-way K split) with x_stride = K + 64 and
    y_stride = M + 8"""
    rng = np.random.default_rng(K + N)
    wq = mx.swept_weights(t, M, K, rng)
    xh = rng.standard_normal((N, K)).astype(np.float16)
    xs = np.full((N, K + 64), np.nan, np.float16)
    xs[:, :K] = xh
    W = gpu.Weight(t, K, M, wq)
    xd, xsd, yd = gpu.DevBuf(src=xh), gpu.DevBuf(src=xs), gpu.DevBuf(N * M * 4)
    assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, yd.ptr, M, 0, impl) == 1
    want = yd.download(np.float32, (N, M))
    assert np.isfinite(want).all()
    ysd = _strided_out(gpu, N, M, M + 8)
    assert gpu.lib().b200_mul_mat_f16(W.h, xsd.ptr, K + 64, N, ysd.ptr, M + 8, 0, impl) == 1
    _check_strided(ysd.download(np.uint32, (N, M + 8)), want, M)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if RATIOS:
        print("\nlargest error / bound per kernel family and shape:")
        for k in sorted(RATIOS):
            print("  %-44s %.3f" % (k, RATIOS[k]))
