"""CPU tests of the exact-arithmetic mat-vec reference (tests/mmv_exact.py) that the GPU mat-vec tests compare against.

  * it agrees, within a bound of the same kind at the CPU's summation depth, with the oracle's mul_mat (ggml's vec_dot order)
  * its bound for the GPU kernels is tight enough to catch the defects a block-quantised mat-vec typically has: a piece that reads
    the neighbouring block's activation scale, a row that drops its last ragged piece or work unit, a block that takes its weight
    scale from the next row, Q4_K mins applied to the wrong half, Q3_K high bits taken from the other half.  Each moves some output
    by at least 10x its bound, so a GPU test that holds a kernel to the bound fails on it.
"""
import numpy as np
import pytest
import pyoracle as po
import mmv_exact as mx

# the loosest reduction of any launch shape: the generic kernel's per-lane chain or the fast kernel's 512 x J4 (depth 23)
FAST_WIDEST = ("fast", 512, 4)


def _loosest_bound(t, wq, K, q, d, s, **kw):
    y, b_gen, mag, _ = mx.reference(t, wq, K, q, d, s, ("generic",), **kw)
    b_fast = mx.gamma(mx.R[t] + mx.depth(t, K, FAST_WIDEST)) * mag
    return y, np.maximum(b_gen, b_fast)


def _case(orc, t, M, K, seed):
    rng = np.random.default_rng(seed)
    wq = mx.swept_weights(t, M, K, rng)
    x = mx.swept_acts(t, 1, K, rng)
    q, d, s, _ = mx.act_from_blocks(t, orc.quantize_act(t, x), K)
    return wq, x, q[0], d[0], s[0]


@pytest.mark.parametrize("K", [1024, 32768])
@pytest.mark.parametrize("t", po.WEIGHT_TYPES)
def test_reference_agrees_with_cpu_mul_mat(orc, t, K):
    """the restatement against orc.mul_mat (quantise_act + vec_dot in the CPU's order) within the CPU's own error bound"""
    M = 24
    wq, x, q, d, s = _case(orc, t, M, K, 1000 * t + K)
    want = orc.mul_mat(t, wq, K, M, x)[0].astype(np.float64)
    y, bound, mag, (A, B) = mx.reference(t, wq, K, q, d, s, ("generic",), rows=np.arange(M))
    lanes = mx.cpu_lane_magnitude(t, wq, K, q, d) if t in (po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K) else None
    cb = mx.cpu_bound(t, K, A, B, lanes)
    err = np.abs(y - want)
    assert np.all(err <= cb), (po.TYPE_NAMES[t], float((err / cb).max()))
    # the restatement is not loose: the sum of |terms| is within a small factor of |w| |x| and the output is far above the bound
    wd = np.abs(orc.dequantize(t, wq, K)).astype(np.float64)
    xdq = np.abs(q.astype(np.float64) * np.repeat(d.astype(np.float64), K // d.size))
    assert np.all(mag <= 1.01 * (wd @ xdq) + 1e-30)
    assert np.median(bound / np.maximum(np.abs(y), 1e-30)) < 1e-4


def _ratio(y_mut, y, bound):
    return float((np.abs(y_mut - y) / bound).max())


# (type, smallest K, largest K) of the GPU test matrix
SENS = [(po.Q4_K, 2048, 65536), (po.Q4_0, 2048, 65536), (po.Q3_K, 8192, 59392), (po.Q5_K, 4608, 32768), (po.Q6_K, 4608, 32768),
        (po.Q5_0, 4544, 32768), (po.Q8_0, 4544, 32768), (po.Q2_K, 4608, 32768), (po.Q4_1, 4544, 32768), (po.Q5_1, 4544, 32768)]
MARGIN = 10.0


@pytest.mark.parametrize("t,K_small,K_large", SENS, ids=[po.TYPE_NAMES[s[0]] for s in SENS])
def test_bound_catches_index_mistakes(orc, t, K_small, K_large):
    """every mutation misses the loosest kernel bound by >= MARGIN x on some output, at the smallest and the largest K"""
    M = 12
    ratios = {}
    for K in (K_small, K_large):
        wq, x, q, d, s = _case(orc, t, M, K, 77 + K)
        y, bound = _loosest_bound(t, wq, K, q, d, s)
        muts = {"piece reads the next block's activation scale": dict(xd_piece=mx.PPB[t] - 1),
                # a piece can nearly cancel (A ~ B) in one row; a kernel that skips the ragged last piece skips it in every row
                "last piece of every row dropped": dict(drop=("piece", None)),
                "last work unit of a row dropped": dict(drop=("unit", 5)),
                "last block's scale from the next row": dict(d_from_next_row=(2, K // mx.BE[t] - 1))}
        if t in (po.Q4_K, po.Q5_K):
            muts["m0 / m1 swapped"] = dict(swap_mins=True)
        if t == po.Q3_K:
            muts["high bit from the other half"] = dict(q3_hbit_other_half=True)
        for what, kw in muts.items():
            ym, _ = _loosest_bound(t, wq, K, q, d, s, **kw)
            ratios[(K, what)] = _ratio(ym, y, bound)
    print(po.TYPE_NAMES[t], {k: round(v, 1) for k, v in ratios.items()})
    low = {k: v for k, v in ratios.items() if v < MARGIN}
    assert not low, low


def test_gelu_window():
    """gelu_ok accepts the LUT value of f16(y) and rejects a neighbouring fp16 output far from any midpoint"""
    y = np.array([0.3, -1.7, 2.5, -0.02], np.float64)
    f = y.astype(np.float16).astype(np.float64)
    g, _ = mx._gelu_outputs(f)
    assert np.all(mx.gelu_ok(g, y, np.full(4, 1e-9)))
    other = np.nextafter(g.astype(np.float16), np.float16(np.inf)).astype(np.float64)
    assert not np.any(mx.gelu_ok(other, y, np.full(4, 1e-9)))
