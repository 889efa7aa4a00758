"""CPU: the weight-quantiser cases (tests/wquant_cases.py) test what they claim, and the oracle writes the reference's blocks on them.

Findings about the reference these tests rest on:

* quantize_row_q{2,4,5}_K_reference carry make_qkx1_quants's codes from block to block inside one call: the oracle restates that,
  and where the compiled reference exists it agrees byte for byte on every case, called once per row.
* ggml_quantize_q{2,4,5}_K(src, dst, n, k) do not quantise rows of k: they loop `for (j = 0; j < nb; j += k)` with nb = k / 256
  (k_quants.c:381-391, 639-648, 768-777), which runs once, so ONE call quantises the first k values and leaves the rest of dst as
  it was.  Called on four rows of 1024 with k = 1024, 12 of 16 blocks are whatever dst held before -- they match no quantiser.
  test_ggml_quantize_k_writes_one_call_of_k pins this.  The model quantiser goes through ggml_quantize_chunk, which passes n as k,
  so there one call, and one chain of codes, spans a whole chunk of 32 * 512 values (or the whole tensor on one thread) across
  row boundaries.  Rows are what the device quantises independently, so the row-by-row call is what it is held to.
"""
import numpy as np
import pytest
import pyoracle as po
import wquant_cases as wc

CASES = wc.cases()
STALE = [c for c in CASES if c.catches]


def _blocks(t, q):
    return q.reshape(-1, po.BLOCK_BYTES[t])


@pytest.mark.parametrize("case", STALE, ids=lambda c: c.name)
def test_stale_cases_reach_the_carried_codes(orc, case):
    """each stale case makes the chained oracle and the fresh-codes oracle differ in some block, for every type it claims"""
    for t in case.catches:
        a, b = orc.quantize(t, case.x), orc.quantize(t, case.x, fresh_codes=True)
        differ = (_blocks(t, a) != _blocks(t, b)).any(axis=1)
        assert differ.any(), (case.name, po.TYPE_NAMES[t])
        nb = case.x.shape[1] // 256
        assert not differ.reshape(-1, nb)[:, 0].any(), (case.name, po.TYPE_NAMES[t])     # block 0 of a row starts from zeros in both


def test_every_chained_type_and_family_is_caught():
    names = {c.name for c in STALE}
    assert {"stale_tiled", "stale_tiled_scaled", "stale_sub32", "stale_sub16", "stale_midrow", "stale_every_second"} <= names
    for c in STALE:
        if c.name != "stale_sub16":
            assert set(c.catches) == set(wc.CHAINED), c.name
    assert po.Q2_K in next(c for c in STALE if c.name == "stale_sub16").catches


def test_cases_avoid_block0_repeats_and_cover_the_shapes():
    """no row's first block repeats the block quantised just before it (the reference reads uninitialised stack there)"""
    for c in CASES:
        x = c.x
        if x.shape[0] > 1 and x.shape[1] >= 256 and np.abs(x).max() > 0 and c.name != "control":
            assert not np.any(np.all(x[1:, :256] == x[:-1, -256:], axis=1)), c.name
    widths = {c.x.shape[1] for c in CASES}
    assert {256, 4544, 8192, 14848} <= widths
    assert any(c.x.shape[0] >= 1024 and c.x.shape[1] <= 512 for c in CASES)
    assert any(c.x.shape[0] == 1 and c.x.shape[1] >= 65536 for c in CASES)
    assert next(c for c in CASES if c.name == "k4544").types == (po.Q4_0,)
    assert all(("ongrid_" + po.TYPE_NAMES[t]) in {c.name for c in CASES} for t in wc.KQUANTS)


def test_fresh_codes_only_touch_the_chained_types(orc):
    c = next(c for c in CASES if c.name == "stale_tiled")
    for t in (po.Q4_0, po.Q3_K, po.Q6_K):
        assert np.array_equal(orc.quantize(t, c.x), orc.quantize(t, c.x, fresh_codes=True))


def test_big_case_rows():
    idx = wc.big_sample_rows()
    assert idx.min() == 0 and idx.max() == wc.BIG_ROWS - 1
    assert wc.BIG_ROWS * wc.BIG_K * 4 > 1 << 31
    edge = (1 << 31) // (wc.BIG_K * 4)
    assert edge in idx and edge + 1 in idx
    r = wc.big_rows(idx)
    assert r.shape == (idx.size, wc.BIG_K) and r.dtype == np.float32
    assert np.array_equal(r[0], wc.big_rows([wc.BIG_POOL * 7])[0])            # r and r + 61 * 7 are the same row


needs_ref = pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref/libggml_ref.so not built (needs the reference sources)")


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_oracle_is_the_reference_row_by_row(orc, case):
    """quantize_row_q*_reference (after ggml_init, which fills its fp16 table) called once per row, byte for byte"""
    ref = po.ref()
    for t in case.types:
        assert np.array_equal(orc.quantize(t, case.x), ref.quantize(t, case.x)), (case.name, po.TYPE_NAMES[t])


@needs_ref
def test_oracle_is_the_reference_on_sampled_big_rows(orc):
    x = wc.big_rows(wc.big_sample_rows()[:6])
    for t in wc.TYPES:
        assert np.array_equal(orc.quantize(t, x), po.ref().quantize(t, x)), po.TYPE_NAMES[t]


@needs_ref
@pytest.mark.parametrize("t", wc.CHAINED)
def test_ggml_quantize_k_writes_one_call_of_k(orc, t):
    """ggml_quantize_q*_K(src, dst, n = 4096, k = 1024) writes the first row's 4 blocks, chained as one call, and nothing else"""
    import ctypes as C
    fn = getattr(po.ref().L, "ggml_quantize_" + po.TYPE_NAMES[t])
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    fn.restype = C.c_size_t
    x = np.tile(np.random.default_rng(3).standard_normal(1024).astype(np.float32), (4, 1))
    bb = po.BLOCK_BYTES[t]
    dst = np.full(16 * bb, 0xA5, np.uint8)
    hist = np.zeros(16, np.int64)
    fn(x.ctypes.data, dst.ctypes.data, x.size, 1024, hist.ctypes.data)
    assert np.array_equal(dst[:4 * bb], orc.quantize(t, x[0]))
    assert (dst[4 * bb:] == 0xA5).all()
