"""-m gpu: the prompt GEMM bit for bit at every producer, token tile and K split, on exactly representable operands (tests/gemm_exact.py).

  * grid-exact: b200_mul_mat_f16 with impl 1 (wgmma) and impl 0 (CUDA core), and b200_mul_mat (activation quantiser + dispatcher,
    N > 512 in chunks, K % 64 == 32 on the CUDA-core kernel): every output equals the fp64 model bit for bit; Y rows are M + 3 apart
    in a buffer with one extra token row, all pre-filled with a NaN sentinel that every gap column and the extra row must keep
  * GELU epilogue: on grid operands the accumulator is exact, so GEMM + GELU equals b200_gelu of the exact values, bit for bit
  * one-hot readback: Y[n][m] = fp16(w[m][k_n]) for every type, on swept, fp16-subnormal and top-binade weights: each producer's one
    rounding to fp16 (Q4_K's fp32 fma, the half arithmetic of Q4_0 / Q3_K, the generic dequantiser)
  * a two-way K split gives the same bits on every run; impl 1 refuses (returns 0, writes nothing) what it does not cover
The (type, producer, BN, ksplit, K blocks per CTA) combinations the module ran are printed at its end (pytest -s).
"""
import collections
import functools
import numpy as np
import pytest
import pyoracle as po
import mmv_exact as mx
import gemm_exact as gx

pytestmark = pytest.mark.gpu
NAN_BITS = np.uint32(0x7FC0DEAD)
REACHED = collections.defaultdict(set)


def _record(c, gelu, what):
    t, K, M, N = c
    for s, n in gx.launches(c, gelu):
        if s is None:
            REACHED[(po.TYPE_NAMES[t], "cuda-core", 0, 0)].add(what)
            continue
        kbs = [kb for _, kb in gx.halves(K, s[1])]
        prod = po.TYPE_NAMES[s[2]] if s[2] >= 0 else "generic"
        REACHED[(po.TYPE_NAMES[t], prod, s[0], s[1])].add("KB %d..%d" % (min(kbs), max(kbs)))


@functools.lru_cache(maxsize=4)
def _grid_case(c, q8=False):
    """-> (weights, activations, exact Y as float32) of a case"""
    t, K, M, N = c
    rng = np.random.default_rng(gx.case_seed(c))
    wq = gx.grid_weights(t, M, K, rng)
    x = gx.grid_acts_q8(t, N, K, rng) if q8 else gx.grid_acts(N, K, rng)
    y, mag = gx.gemm_model(t, wq, K, x, mag=True)
    assert mag.max() <= gx.HEADROOM * gx.G, mag.max() / gx.G
    y32 = y.astype(np.float32)
    assert np.array_equal(y32.astype(np.float64), y)
    return wq, x, y32


def _sentinel_y(gpu, N, M):
    return gpu.DevBuf(src=np.full((N + 1, M + 3), NAN_BITS, np.uint32))


def _check(got, want, c, what):
    """got: uint32 [N + 1][M + 3] bits, want: float32 [N][M]"""
    t, K, M, N = c
    bad = np.argwhere(got[:N, :M] != want.view(np.uint32))
    if bad.size:
        n, m = bad[0]
        pytest.fail("%s %s: %d outputs differ; first at token %d row %d: got %r want %r (launches %s)" % (
            gx.case_id(c), what, len(bad), n, m, got[n, m:m + 1].view(np.float32)[0], want[n, m], gx.launches(c)))
    assert np.all(got[:N, M:] == NAN_BITS), (what, "gap columns written", int((got[:N, M:] != NAN_BITS).sum()))
    assert np.all(got[N] == NAN_BITS), (what, "extra token row written")


def _f16_call(gpu, W, x, c, impl, gelu):
    t, K, M, N = c
    xd, yd = gpu.DevBuf(src=np.ascontiguousarray(x, np.float16)), _sentinel_y(gpu, N, M)
    assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, yd.ptr, M + 3, gelu, impl) == 1
    return yd.download(np.uint32, (N + 1, M + 3))


@pytest.mark.parametrize("impl", [1, 0], ids=["wgmma", "cuda_core"])
@pytest.mark.parametrize("c", gx.TC, ids=gx.case_id)
def test_grid_exact(gpu, c, impl):
    t, K, M, N = c
    wq, x, want = _grid_case(c)
    W = gpu.Weight(t, K, M, wq)
    _check(_f16_call(gpu, W, x, c, impl, 0), want, c, "impl %d" % impl)
    if impl == 1:
        _record(c, False, "grid")


@pytest.mark.parametrize("c", gx.MUL_MAT, ids=gx.case_id)
def test_grid_exact_dispatcher(gpu, orc, c):
    """b200_mul_mat: the rows quantise to themselves (test_gemm_exact.py), so the chunked GEMM must give the exact product"""
    t, K, M, N = c
    wq, x, want = _grid_case(c, q8=True)
    W, xd, yd = gpu.Weight(t, K, M, wq), gpu.DevBuf(src=x), _sentinel_y(gpu, N, M)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, N, yd.ptr, M + 3)
    _check(yd.download(np.uint32, (N + 1, M + 3)), want, c, "b200_mul_mat")
    _record(c, False, "dispatcher")


@pytest.mark.parametrize("impl", [1, 0], ids=["wgmma", "cuda_core"])
@pytest.mark.parametrize("c", gx.GELU, ids=gx.case_id)
def test_grid_exact_gelu_epilogue(gpu, c, impl):
    t, K, M, N = c
    wq, x, y = _grid_case(c)
    yd, gd = gpu.DevBuf(src=y), gpu.DevBuf(y.nbytes)
    gpu.lib().b200_gelu(yd.ptr, gd.ptr, y.size)
    want = gd.download(np.float32, y.shape)
    W = gpu.Weight(t, K, M, wq)
    _check(_f16_call(gpu, W, x, c, impl, 1), want, c, "GELU impl %d" % impl)
    if impl == 1:
        _record(c, True, "gelu")


# ------------------------------------------------------------------------------------------------ one-hot readback
def _edge_weights(orc, t, M, K, rng):
    """swept_weights, with rows M-4, M-3 scaled into the fp16 subnormal range and rows M-2, M-1 into the top binade (<= 65504)"""
    if t == po.F16:
        w = rng.standard_normal((M, K)) * np.exp2(rng.uniform(-12, 2, (M, 1)))
        w[M - 4:M - 2] = rng.standard_normal((2, K)) * np.exp2(rng.uniform(-26, -14, (2, K)))
        w[M - 2:] = rng.uniform(-65504, 65504, (2, K))
        w[M - 2:, :4] = [65504, -65504, 65488, -32768]
        return w.astype(np.float16)
    wq = mx.swept_weights(t, M, K, rng)
    nb, bb = K // mx.BE[t], po.BLOCK_BYTES[t]
    v = wq.reshape(M, nb, bb)
    fields = [mx.D_OFF[t]] + ([mx.M_OFF[t]] if t in mx.M_OFF else [])
    for off in fields:                                     # positive fp16 subnormal scales (Q4_1 / Q5_1 m: either sign)
        bits = rng.integers(1, 0x40, (2, nb)).astype(np.uint16)       # d <= 63 * 2^-24
        if t in (po.Q4_1, po.Q5_1) and off == 2:
            bits |= (rng.integers(0, 2, (2, nb)) << 15).astype(np.uint16)
        v[M - 4:M - 2, :, off:off + 2] = bits[..., None].view(np.uint8)
    w = orc.dequantize(t, v[M - 2:].reshape(2, -1), K).astype(np.float64).reshape(2, nb, -1)
    amax = np.abs(w).max(-1)
    e = np.where(amax > 0, np.floor(np.log2(65504.0 / np.where(amax > 0, amax, 1))), 0)
    for off in fields:                                     # a power of two scales every fp32 value of the block exactly
        f = v[M - 2:, :, off:off + 2].copy().view(np.float16)[..., 0].astype(np.float64)
        v[M - 2:, :, off:off + 2] = (f * np.exp2(e)).astype(np.float16)[..., None].view(np.uint8)
    return v.reshape(M, -1)


def _onehot_columns(K, N, ks):
    """every column, or (for long rows) the first two, the last two and the two K blocks around each split boundary"""
    kbt = K // gx.BK
    if kbt * gx.BK <= 48 * N:
        return np.arange(K)
    kbs = {0, 1, kbt - 2, kbt - 1} | {b for kb0, _ in gx.halves(K, ks) for b in (kb0 - 1, kb0) if 0 <= b < kbt}
    return np.concatenate([np.arange(b * gx.BK, (b + 1) * gx.BK) for b in sorted(kbs)])


ONEHOT = [c for c in gx.TC if c[2] <= 1024]


@pytest.mark.parametrize("c", ONEHOT, ids=gx.case_id)
def test_tensor_core_gemm_operand_is_the_exact_fp16_weight(gpu, orc, c):
    """One-hot activation rows read the dequantised A operand back: Y[n][m] = fp16(w[m][k_n]) exactly, on both kernels.  Pins the
    per-type dequantisation producers of gemm_tc.cu (Q4_K fp32 fma; Q4_0 / Q3_K half arithmetic; generic for the rest) to
    dequantize_row_* + one fp16 rounding, subnormal results and the top binade included (values past 65504 are not used: inf x 0
    would turn the whole row into NaN)"""
    t, K, M, N = c
    rng = np.random.default_rng(gx.case_seed(c) + 1)
    wq = _edge_weights(orc, t, M, K, rng)
    wf = (np.asarray(wq, np.float16) if t == po.F16 else orc.dequantize(t, wq, K)).astype(np.float16)
    assert np.isfinite(wf).all()
    sub = (wf[M - 4:M - 2] != 0) & (np.abs(wf[M - 4:M - 2]) < np.float16(2.0 ** -14))
    assert sub.any(axis=1).all()                                                         # both tiny rows reach subnormal values
    assert np.all(np.abs(wf[M - 2:].astype(np.float32)).max(1) >= 32768)                 # both huge rows reach the top binade
    want = wf.astype(np.float32) + np.float32(0)          # the accumulators start at +0, and +0 + -0 = +0: a -0 weight reads back as +0
    W = gpu.Weight(t, K, M, wq)
    (s, _), = gx.launches(c)
    cols = _onehot_columns(K, N, s[1] if s else 1)
    for off in range(0, len(cols), N):
        cc = cols[off:off + N]
        xh = np.zeros((N, K), np.float16)
        xh[np.arange(len(cc)), cc] = 1.0
        xd, yd = gpu.DevBuf(src=xh), gpu.DevBuf(N * M * 4)
        for impl in (1, 0):
            assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, yd.ptr, M, 0, impl) == 1
            got = yd.download(np.float32, (N, M))[:len(cc)]
            bad = np.argwhere(got.view(np.uint32) != want[:, cc].T.view(np.uint32))
            if bad.size:
                (i, m), k = bad[0], cc[bad[0][0]]
                pytest.fail("%s impl %d: %d weights read back wrong; first at row %d column %d: got %r (0x%08x) want %r (0x%08x)" % (
                    gx.case_id(c), impl, len(bad), m, k, got[i, m], got[i:i + 1, m].view(np.uint32)[0], want[m, k],
                    want[m:m + 1, k].view(np.uint32)[0]))
    _record(c, False, "one-hot")


# ------------------------------------------------------------------------------------------------ determinism and refusals
@pytest.mark.parametrize("t,K,M,N", [(po.Q4_K, 8192, 300, 512), (po.Q4_0, 4544, 200, 40), (po.Q5_K, 14848, 129, 100)])
def test_k_split_is_deterministic(gpu, t, K, M, N):
    """ksplit == 2 adds two partial tiles into a zeroed Y: 0 + a + b is the same in either order, so random (non-grid) data gives the
    same bits on every run"""
    import ggllm_cpp_b200.ggcc as ggcc
    assert gx.launches((t, K, M, N))[0][0][1] == 2
    rng = np.random.default_rng(K + M + N)
    W = gpu.Weight(t, K, M, ggcc.random_blocks(t, M, K, rng))
    xd, yd = gpu.DevBuf(src=rng.standard_normal((N, K)).astype(np.float16)), gpu.DevBuf(N * M * 4)
    runs = []
    for _ in range(3):
        assert gpu.lib().b200_mul_mat_f16(W.h, xd.ptr, K, N, yd.ptr, M, 0, 1) == 1
        runs.append(yd.download(np.uint32, (N, M)))
    assert np.isfinite(runs[0].view(np.float32)).all()
    assert np.array_equal(runs[0], runs[1]) and np.array_equal(runs[0], runs[2])


def test_tensor_core_gemm_refuses_uncovered_operands(gpu):
    """impl 1 returns 0 and writes nothing for x_stride % 8 != 0, for an x that is not 16-byte aligned, for N > 512 and K % 64 != 0"""
    t, K, M, N = po.Q4_K, 1024, 130, 40
    rng = np.random.default_rng(5)
    W = gpu.Weight(t, K, M, gx.grid_weights(t, M, K, rng))
    xd = gpu.DevBuf(src=gx.grid_acts(600, K + 8, rng))
    yd = _sentinel_y(gpu, 600, M)
    for x_ptr, xs, n in ((xd.ptr, K + 4, N), (xd.ptr + 2, K + 8, N), (xd.ptr + 8, K + 8, N), (xd.ptr, K, 513)):
        assert gpu.lib().b200_mul_mat_f16(W.h, x_ptr, xs, n, yd.ptr, M + 3, 0, 1) == 0
    W2 = gpu.Weight(po.Q4_0, K - 32, M, gx.grid_weights(po.Q4_0, M, K - 32, rng))
    assert gpu.lib().b200_mul_mat_f16(W2.h, xd.ptr, K, N, yd.ptr, M + 3, 0, 1) == 0
    gpu.lib().b200_synchronize()
    assert np.all(yd.download(np.uint32, (601, M + 3)) == NAN_BITS)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REACHED:
        print("\n(type, producer, BN, ksplit) reached, K blocks per CTA:")
        for k in sorted(REACHED):
            print("  %-6s %-9s BN %3d  ksplit %d   %s" % (k + (", ".join(sorted(REACHED[k])),)))
