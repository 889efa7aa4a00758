"""-m gpu: the host twin of tests/device_random.py against what the device writes.

  * b200_weight_random for every weight type: b200_dequantize_rows of the device planes equals orc.dequantize of the twin's blocks
    bit for bit (F16 / F32: the twin's values) -- at a small shape, at K = 4544 (Q4_0 rows of 142 blocks, not a multiple of 16 bytes
    in the scale plane) and on the 65024 x 8192 Q4_K head of Falcon-40B (first rows, last rows and a spread between them, where the
    block index times 8 shifted by 20 is far past 2^32).
  * b200_falcon_kv_fill_random into an f32 and an fp16 cache at pos > 0: kv_read of rows [pos, pos + n) equals the twin, every other
    row keeps what was there."""
import numpy as np
import pytest
import pyoracle as po
import device_random as dr
from helpers import TINY_40B

pytestmark = pytest.mark.gpu


def _check_rows(gpu, orc, t, K, M, rows, seed):
    W = gpu.Weight(t, K, M, seed=seed)
    try:
        got = W.dequantize(rows)
    finally:
        W.free()
    twin = dr.weight_rows(t, K, rows, seed)
    want = twin.astype(np.float32) if t in (po.F32, po.F16) else orc.dequantize(t, twin, K)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, "%s K %d: %d values differ, first (row, k) %s" % (po.TYPE_NAMES[t], K, len(bad), bad[:1].tolist())


@pytest.mark.parametrize("t", dr.TYPES)
def test_weight_random_small(gpu, orc, t):
    K = 512 if dr.TYPE_SPEC[t][0] == 256 else 96
    _check_rows(gpu, orc, t, K, 37, np.arange(37), seed=1234 * 1000003 + 7)


def test_weight_random_falcon7b_width(gpu, orc):
    _check_rows(gpu, orc, po.Q4_0, 4544, 300, np.arange(300), seed=55)


def test_weight_random_falcon40b_head(gpu, orc):
    M = 65024
    rows = np.unique(np.concatenate([np.arange(8), np.arange(M - 8, M), np.linspace(0, M - 1, 97).astype(np.int64)]))
    _check_rows(gpu, orc, po.Q4_K, 8192, M, rows, seed=1234 * 1000003 + 483)


@pytest.mark.parametrize("kv_f16", [False, True])
def test_kv_fill_random(gpu, kv_f16):
    hp = dict(TINY_40B)
    n_ctx, pos, n = 64, 13, 29
    f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=1, kv_f16=kv_f16)
    try:
        w = hp["n_head_kv"] * (hp["n_embd"] // hp["n_head"])
        rng = np.random.default_rng(3)
        for l in range(hp["n_layer"]):
            f.kv_write(l, 0, rng.standard_normal((n_ctx, w)).astype(np.float32), rng.standard_normal((n_ctx, w)).astype(np.float32))
        before = [f.kv_read(l, 0, n_ctx) for l in range(hp["n_layer"])]
        f.kv_fill_random(pos, n, seed=77)
        for l in range(hp["n_layer"]):
            k, v = f.kv_read(l, 0, n_ctx)
            kt, vt = dr.kv_rows(l, pos, n, w, seed=77, f16=kv_f16)
            assert np.array_equal(k[pos:pos + n].view(np.uint32), kt.view(np.uint32)), ("K", l)
            assert np.array_equal(v[pos:pos + n].view(np.uint32), vt.view(np.uint32)), ("V", l)
            out = np.ones(n_ctx, bool)
            out[pos:pos + n] = False
            assert np.array_equal(k[out], before[l][0][out]) and np.array_equal(v[out], before[l][1][out]), ("outside rows", l)
    finally:
        f.free()
