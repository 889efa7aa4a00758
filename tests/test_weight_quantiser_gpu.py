"""GPU: b200_quantize_weights_rows on every case of tests/wquant_cases.py, for every type with a device quantiser, byte for byte against
the oracle called once per row (which is the reference's quantize_row_q*_reference, tests/test_wquant_cases.py).

The stale-code cases make Q2_K / Q4_K / Q5_K's fits start from the previous block's codes; a quantiser that starts every block from
fresh codes gets them wrong.  Quantising the same buffer twice must give the same bytes (no uninitialised state), and every block
must dequantise on the device to the oracle's values (NaNs from fp16-overflowing scales compare as NaN, not by payload)."""
import numpy as np
import pytest
import pyoracle as po
import wquant_cases as wc

pytestmark = pytest.mark.gpu

CASES = wc.cases()
FIELDS = {po.Q4_0: [("d", 0, 2), ("qs", 2, 18)],
          po.Q2_K: [("scales", 0, 16), ("qs", 16, 80), ("d", 80, 82), ("dmin", 82, 84)],
          po.Q3_K: [("hmask", 0, 32), ("qs", 32, 96), ("scales", 96, 108), ("d", 108, 110)],
          po.Q4_K: [("d", 0, 2), ("dmin", 2, 4), ("scales", 4, 16), ("qs", 16, 144)],
          po.Q5_K: [("d", 0, 2), ("dmin", 2, 4), ("scales", 4, 16), ("qh", 16, 48), ("qs", 48, 176)],
          po.Q6_K: [("ql", 0, 128), ("qh", 128, 192), ("scales", 192, 208), ("d", 208, 210)]}


def _first_difference(t, got, want, K):
    """'row r block b field f' of the first differing block, and how many blocks differ"""
    bb, nb = po.BLOCK_BYTES[t], K // po.BLOCK_ELEMS[t]
    g, w = got.reshape(-1, bb), want.reshape(-1, bb)
    bad = np.flatnonzero((g != w).any(axis=1))
    if bad.size == 0:
        return None
    i = int(bad[0])
    fields = [f for f, lo, hi in FIELDS[t] if not np.array_equal(g[i, lo:hi], w[i, lo:hi])]
    return "%s: %d of %d blocks differ; first: row %d block %d, fields %s" % (
        po.TYPE_NAMES[t], bad.size, g.shape[0], i // nb, i % nb, ",".join(fields))


def _quantise(gpu, t, x, times=1):
    K = x.shape[1]
    xd, out = gpu.DevBuf(src=x), gpu.DevBuf(x.shape[0] * po.row_bytes(t, K))
    res = []
    for _ in range(times):
        out.upload(np.full(out.nbytes, 0x5A, np.uint8))                   # nothing may survive from a previous call
        assert gpu.lib().b200_quantize_weights_rows(t, xd.ptr, out.ptr, x.size, K) == 1
        res.append(out.download(np.uint8, (x.shape[0], po.row_bytes(t, K))))
    xd.free(), out.free()
    return res


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_device_blocks_are_the_oracle_blocks(gpu, orc, case):
    errors = []
    for t in case.types:
        want = orc.quantize(t, case.x)
        got, again = _quantise(gpu, t, case.x, times=2)
        diff = _first_difference(t, got, want, case.x.shape[1])
        if diff:
            errors.append(diff)
        elif not np.array_equal(got, again):
            errors.append("%s: a second run over the same buffer wrote other bytes" % po.TYPE_NAMES[t])
        else:                                                           # the device dequantiser reads them as the oracle does
            w = gpu.Weight(t, case.x.shape[1], case.x.shape[0], blocks=got)
            deq = w.dequantize()
            w.free()
            ref = orc.dequantize(t, want, case.x.shape[1])
            if not np.array_equal(deq, ref, equal_nan=True):            # the 1e8 row overflows fp16 scales: NaN payloads differ
                errors.append("%s: dequantised blocks differ from the oracle's" % po.TYPE_NAMES[t])
    assert not errors, "%s: %s" % (case.name, "; ".join(errors))


def test_big_matrix_sampled_rows(gpu, orc):
    """65024 x 14848 fp32 (3.9 GB, past 2^31 bytes): every type, sampled rows against the oracle, the rest finite-length checked"""
    x = wc.big_matrix()
    idx = wc.big_sample_rows()
    xs = x[idx]
    xd = gpu.DevBuf(src=x)
    del x
    errors = []
    for t in wc.TYPES:
        rb = po.row_bytes(t, wc.BIG_K)
        out = gpu.DevBuf(wc.BIG_ROWS * rb)
        assert gpu.lib().b200_quantize_weights_rows(t, xd.ptr, out.ptr, wc.BIG_ROWS * wc.BIG_K, wc.BIG_K) == 1
        got = out.download(np.uint8, (wc.BIG_ROWS, rb))[idx]
        out.free()
        diff = _first_difference(t, got, orc.quantize(t, xs), wc.BIG_K)
        if diff:
            errors.append(diff + " (rows are indices into %s)" % list(idx))
    xd.free()
    assert not errors, errors


def test_return_codes(gpu):
    x = np.random.default_rng(5).standard_normal((2, 512)).astype(np.float32)
    xd, out = gpu.DevBuf(src=x), gpu.DevBuf(2 * po.row_bytes(po.Q5_K, 512))
    q = gpu.lib().b200_quantize_weights_rows
    for t in wc.TYPES:
        qk = po.BLOCK_ELEMS[t]
        assert q(t, xd.ptr, out.ptr, 0, 512) == 1                      # nothing to do, nothing launched
        assert q(t, xd.ptr, out.ptr, 512 + qk // 2, 512) == -1         # n_elems not a multiple of the row
        assert q(t, xd.ptr, out.ptr, 480, 480) == (-1 if qk == 256 else 1)
        assert q(t, xd.ptr, out.ptr, 1024, 512 + qk // 2) == -1        # row not a multiple of the block
        assert q(t, xd.ptr, out.ptr, 1024, 0) == -1
        assert q(t, xd.ptr, out.ptr, -512, 512) == -1
    for t in (po.F32, po.F16, po.Q4_1, po.Q5_0, po.Q5_1, po.Q8_0, po.Q8_K, 99):
        assert q(t, xd.ptr, out.ptr, 1024, 512) == 0                   # no device quantiser: the caller quantises on the host
    gpu.lib().b200_synchronize()
    xd.free(), out.free()


@pytest.mark.parametrize("name", ["stale_tiled", "stale_every_second", "many_rows"])
def test_whole_buffer_is_one_row(gpu, orc, name):
    """b200_quantize_weights: the buffer as one row, the codes carried across what were row boundaries (one call of
    quantize_row_q*_reference over all of it, as ggml_quantize_chunk makes)"""
    x = next(c for c in CASES if c.name == name).x.reshape(1, -1)
    for t in wc.TYPES:
        want = orc.quantize(t, x)
        xd, out = gpu.DevBuf(src=x), gpu.DevBuf(want.nbytes)
        assert gpu.lib().b200_quantize_weights(t, xd.ptr, out.ptr, x.size) == 1
        got = out.download(np.uint8, want.shape)
        xd.free(), out.free()
        diff = _first_difference(t, got, want, x.shape[1])
        assert diff is None, "%s: %s" % (name, diff)
    assert gpu.lib().b200_quantize_weights(po.Q4_K, None, None, 0) == 1
    assert gpu.lib().b200_quantize_weights(po.Q4_K, None, None, 300) == -1
    assert gpu.lib().b200_quantize_weights(po.Q8_0, None, None, 256) == 0
