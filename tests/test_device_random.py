"""The host twin of the device's synthetic data (tests/device_random.py) against a host model of the upload's repack.

The GPU side (test_device_random_gpu.py) holds the twin to b200_weight_random and b200_falcon_kv_fill_random byte for byte; these
tests hold it to itself: the twin's blocks, repacked the way repack_kernel does (unpack_sm6, q3_scale), give back the planes the twin
generated, its rows do not depend on which other rows are built, and its values have the ranges fill_random_kernel promises."""
import numpy as np
import pytest
import pyoracle as po
import device_random as dr


@pytest.mark.parametrize("t", dr.TYPES)
def test_blocks_repack_to_the_generated_planes(t):
    """the twin inverts repack_kernel exactly: every plane byte survives blocks -> planes, including rows whose block index passes
    2^32 >> 23 (idx * 8 + p shifted by 20 leaves 32 bits from block 512 on)"""
    per = dr.TYPE_SPEC[t][0]
    K = 4 * 256 if per == 256 else 256
    rows = np.array([0, 1, 7, 1000, 65023])
    planes = dr.weight_planes(t, K, rows, seed=1234 * 1000003 + 5)
    blocks = dr.planes_to_blocks(t, planes)
    assert blocks.shape == (len(rows), dr.row_bytes(t, K))
    back = dr.blocks_to_planes(t, blocks)
    for p, (a, b) in enumerate(zip(planes, back)):
        assert np.array_equal(a, b), "plane %d" % p


@pytest.mark.parametrize("t", dr.TYPES)
def test_rows_are_row_local(t):
    """a subset of rows equals the same rows of the whole matrix, and different seeds give different bytes"""
    per = dr.TYPE_SPEC[t][0]
    K = 512 if per == 256 else 96
    full = dr.weight_rows(t, K, np.arange(40), seed=77)
    sub = dr.weight_rows(t, K, np.array([3, 39, 17]), seed=77)
    assert np.array_equal(sub.view(np.uint8), full[[3, 39, 17]].view(np.uint8))
    assert not np.array_equal(dr.weight_rows(t, K, np.arange(40), seed=78).view(np.uint8), full.view(np.uint8))


@pytest.mark.parametrize("t", dr.TYPES)
def test_value_ranges(t, orc):
    """F16 / F32 elements are dsm * 10 - 0.02, about [0, 0.04); quantised blocks carry fp16 scales d in [unit, 3 unit), 6-bit sub-scales in
    range, and dequantise to finite values"""
    per = dr.TYPE_SPEC[t][0]
    K = 1024 if per == 256 else 320
    w = dr.weight_rows(t, K, np.arange(64), seed=4321)
    if t in (dr.F32, dr.F16):
        v = w.astype(np.float64)
        assert v.min() >= -1e-8 and v.max() <= 0.04 * (1 + 2 ** -10)            # fp16 may round up to the edge
        return
    planes = dr.weight_planes(t, K, np.arange(64), seed=4321)
    unit = 1e-4 if per == 256 else 2e-3
    for p, off, which in dr.SCALE_FIELDS[t]:
        d = planes[p][..., off:off + 2].copy().view(np.float16).astype(np.float64)
        lo, hi = (unit, 3 * unit) if which == "d" else (4 * unit, 12 * unit)
        assert d.min() >= lo * (1 - 2 ** -10) and d.max() <= hi * (1 + 2 ** -10)
    for (_, _, kind), pl in zip(dr.TYPE_SPEC[t][2], planes):
        if kind == 1:
            assert pl.max() < 64
        if kind == 2:
            s = pl.view(np.int8)
            assert s.min() >= -32 and s.max() < 32
    assert np.isfinite(orc.dequantize(t, w, K)).all()


def test_fill_values():
    """fill_kernel: the fp16 cache holds the f32 values rounded; LayerNorm gamma / beta stay in [1 - 0.1, 1 + 0.1) / [-0.01, 0.01)"""
    k32, v32 = dr.kv_rows(3, 100, 5, 512, seed=77)
    k16, v16 = dr.kv_rows(3, 100, 5, 512, seed=77, f16=True)
    assert np.array_equal(k16, k32.astype(np.float16).astype(np.float32)) and np.array_equal(v16, v32.astype(np.float16).astype(np.float32))
    assert not np.array_equal(k32, v32) and np.abs(k32).max() < 1
    g = dr.layernorm_vector("transformer.ln_f.weight", 8192, 5)
    b = dr.layernorm_vector("transformer.ln_f.bias", 8192, 6)
    assert g.min() >= 0.9 and g.max() < 1.1 and np.abs(b).max() <= 0.01


def test_seeds_follow_set_random():
    """tensor i of falcon_shapes gets seed * 1000003 + i, in that order"""
    from helpers import ggcc
    hp = dict(n_vocab=64, n_embd=64, n_head=1, n_head_kv=1, n_layer=2, falcon_type=40)
    seeds = dr.tensor_seeds(ggcc.falcon_shapes(hp), 1234)
    names = list(ggcc.falcon_shapes(hp))
    assert seeds[names[0]] == 1234 * 1000003 and seeds[names[-1]] == 1234 * 1000003 + len(names) - 1
    assert po.Q4_K == dr.Q4_K and po.Q3_K == dr.Q3_K and po.F16 == dr.F16
