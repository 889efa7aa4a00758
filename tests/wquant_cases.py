"""Input matrices for the device weight quantisers (b200_quantize_weights_rows): fp32 [rows][K], each with the reason it exists.

The quantisers must write, for every row, the blocks quantize_row_q*_reference writes when it is called once on that row.  Random
rows are the easy part.  What goes wrong is state: make_qkx1_quants (the (scale, min) fit of Q2_K, Q4_K and Q5_K) stops refining
after a round that leaves its code buffer L unchanged, and its round 0 compares against what L already holds -- the reference
declares L once per call, so block b of a row starts from block b-1's final codes.  Whenever a sub-block's round-0 codes equal
the codes the same sub-block ended with 256 values earlier, the reference stops after round 0 where fresh codes would refine
further.  On i.i.d. data that practically never happens; on a row whose blocks repeat it happens almost always.  The "stale"
cases below are built for it, and tests/test_wquant_cases.py proves each one reaches it (the chained and the fresh-codes oracle
disagree on at least one of its blocks) for the types listed in its `catches`.

Block 0 of a row is quantised from whatever the reference's stack held (undefined behaviour); the oracle and the device start
it from zeros.  So no case lets block 0 of a row repeat anything: every row's first block is new random data.

  control      the ten rows the first device-quantiser test used: normal, tiny, huge, zero, constant, one-sided, cos, sparse
  stale        a 256-block tiled along the row; tiled with copies scaled by 2 and 0.5 (exact, so the round-0 codes are the same);
               one repeated 32-value (16-value for Q2_K) sub-block at every position j; a repeat that starts mid-row after random
               blocks; blocks that repeat every second block
  on-grid      a row dequantised from each K-type, quantised again (what re-quantising a dequantised model does)
  shapes       K = 256 (one block per row), K = 4544 (Falcon-7B width, Q4_0 only), the Falcon widths 8192 and 14848, many rows
               of few blocks, one row of many blocks
  big          65024 x 14848 (the Falcon-180B lm_head): 3.9 GB of fp32, past 2^31 bytes, so the input offsets need 64 bits;
               built from a row pool so that sampled rows can be rebuilt on the host (big_rows())
"""
import numpy as np
import pyoracle as po

F32 = np.float32
TYPES = (po.Q4_0, po.Q2_K, po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K)
CHAINED = (po.Q2_K, po.Q4_K, po.Q5_K)                 # the types whose fit reads the previous block's codes
KQUANTS = (po.Q2_K, po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K)


class Case:
    def __init__(self, name, x, reason, catches=(), types=TYPES):
        self.name, self.x, self.reason = name, np.ascontiguousarray(x, dtype=F32), reason
        self.catches = tuple(catches)                 # chained types on which this case makes fresh codes differ from chained ones
        self.types = tuple(t for t in types if self.x.shape[1] % po.BLOCK_ELEMS[t] == 0)

    def __repr__(self):
        return "Case(%s, %dx%d)" % (self.name, *self.x.shape)


def _control(K=4096, seed=0):
    rng = np.random.default_rng(seed)
    rows = [rng.standard_normal(K), 1e-8 * rng.standard_normal(K), 1e8 * rng.standard_normal(K), np.zeros(K), np.full(K, 0.37),
            np.abs(rng.standard_normal(K)), -np.abs(rng.standard_normal(K)), 0.1 + 2.0 * np.cos(np.arange(K)),
            0.02 * rng.standard_normal(K), rng.standard_normal(K) * (rng.random(K) < 0.05)]
    return np.stack(rows).astype(F32)


def _catching_block(orc, rng):
    """a random 256-block that, tiled, makes fresh codes differ from chained ones for each of Q2_K, Q4_K and Q5_K.  About one
    random block in four does it for Q5_K, whose 32 levels rarely end where round 0 starts; drawing until one does keeps a
    four-row case from missing Q5_K by chance."""
    while True:
        blk = rng.standard_normal(256).astype(F32)
        row = np.tile(blk, 2)[None]
        if all(not np.array_equal(orc.quantize(t, row), orc.quantize(t, row, fresh_codes=True)) for t in CHAINED):
            return blk


def _tiled(rng, rows, K, scales=(1.0,), first=None):
    """row r: its own random 256-block (row 0: `first` if given), copy i scaled by scales[i % len(scales)] (powers of two: exact)"""
    out = np.empty((rows, K), F32)
    for r in range(rows):
        blk = rng.standard_normal(256).astype(F32)
        if r == 0 and first is not None:
            blk = first
        for b in range(K // 256):
            out[r, 256 * b:256 * (b + 1)] = blk * F32(scales[b % len(scales)])
    return out


def _repeat_sub(rng, n, K):
    """row j: random, except that the n-value sub-block at position j is the same in every block"""
    out = rng.standard_normal((256 // n, K)).astype(F32)
    for j in range(256 // n):
        sub = rng.standard_normal(n).astype(F32)
        for b in range(K // 256):
            out[j, 256 * b + n * j:256 * b + n * (j + 1)] = sub
    return out


def _repeat_from(rng, rows, K, start, first=None):
    """random blocks 0..start-1, then block `start` (row 0: `first` if given) tiled to the row's end"""
    out = rng.standard_normal((rows, K)).astype(F32)
    if first is not None:
        out[0, 256 * start:256 * (start + 1)] = first
    for r in range(rows):
        for b in range(start + 1, K // 256):
            out[r, 256 * b:256 * (b + 1)] = out[r, 256 * start:256 * (start + 1)]
    return out


def _every_second(rng, rows, K):
    """odd blocks are copies of the block before them; even blocks are new"""
    out = rng.standard_normal((rows, K)).astype(F32)
    for b in range(1, K // 256, 2):
        out[:, 256 * b:256 * (b + 1)] = out[:, 256 * (b - 1):256 * b]
    return out


def _on_grid(orc, t, rng, rows, K):
    x = rng.standard_normal((rows, K)).astype(F32)
    return orc.dequantize(t, orc.quantize(t, x), K)


def cases(orc=None):
    """every case but the big one, small enough to run through the oracle in seconds"""
    orc = orc or po.orc()
    rng = np.random.default_rng(20261018)
    cs = [Case("control", _control(), "the ten rows of the first device-quantiser test: normal, tiny, huge, zero, constant, "
                                      "one-sided, cos, sparse")]
    blk = _catching_block(orc, rng)
    cs.append(Case("stale_tiled", _tiled(rng, 4, 4096, first=blk), "one random 256-block per row, tiled: every block after the first "
                   "starts from its own codes", catches=CHAINED))
    cs.append(Case("stale_tiled_scaled", _tiled(rng, 4, 4096, (1.0, 2.0, 0.5), first=_catching_block(orc, rng)), "a tiled block with copies scaled by 2 and "
                   "0.5: the same round-0 codes at another scale", catches=CHAINED))
    cs.append(Case("stale_sub32", _repeat_sub(rng, 32, 8192), "row j repeats its 32-value sub-block j in every block: one Q4_K / "
                   "Q5_K fit per block sees stale codes", catches=CHAINED))
    cs.append(Case("stale_sub16", _repeat_sub(rng, 16, 8192), "row j repeats its 16-value sub-block j in every block: one Q2_K "
                   "fit per block sees stale codes", catches=(po.Q2_K,)))
    cs.append(Case("stale_midrow", _repeat_from(rng, 4, 8192, 13, first=_catching_block(orc, rng)), "13 random blocks, then block 13 tiled to the row's end",
                   catches=CHAINED))
    cs.append(Case("stale_every_second", _every_second(rng, 4, 8192), "each odd block repeats the even block before it",
                   catches=CHAINED))
    for t in KQUANTS:
        cs.append(Case("ongrid_" + po.TYPE_NAMES[t], _on_grid(orc, t, rng, 4, 4096), "rows dequantised from %s, quantised again"
                       % po.TYPE_NAMES[t]))
    cs.append(Case("k256", rng.standard_normal((16, 256)), "one block per row: the chain starts and ends in one block"))
    cs.append(Case("k4544", rng.standard_normal((4, 4544)), "the Falcon-7B width: Q4_0 only, 142 blocks per row"))
    cs.append(Case("k8192", rng.standard_normal((4, 8192)), "the Falcon-40B width"))
    cs.append(Case("k14848", rng.standard_normal((2, 14848)), "the Falcon-180B width, 58 K-blocks per row"))
    cs.append(Case("many_rows", _tiled(rng, 2048, 512), "2048 rows of two blocks, each row a tiled block: more rows than one "
                   "CTA covers, and each row's chain must restart at zero", catches=CHAINED))
    cs.append(Case("one_long_row", _tiled(rng, 1, 65536, (1.0, 2.0), first=_catching_block(orc, rng)), "one row of 256 blocks, a tiled block alternately "
                   "scaled by 2", catches=CHAINED))
    return cs


# ----------------------------------------------------------------------------------------------------------- big
BIG_ROWS, BIG_K, BIG_POOL = 65024, 14848, 61


def _big_pool():
    rng = np.random.default_rng(65024)
    return rng.standard_normal((BIG_POOL, BIG_K)).astype(F32)


def big_rows(idx, pool=None):
    """rows idx of the big matrix: pool row r % 61 (so neighbouring rows differ) scaled by 1 + (r % 7) / 8 (exact in fp32)"""
    pool = _big_pool() if pool is None else pool
    idx = np.asarray(idx, np.int64)
    return pool[idx % BIG_POOL] * (F32(1) + (idx % 7).astype(F32)[:, None] / F32(8))


def big_matrix():
    """the whole 65024 x 14848 matrix (3.9 GB)"""
    pool, out = _big_pool(), np.empty((BIG_ROWS, BIG_K), F32)
    for r0 in range(0, BIG_ROWS, 4096):
        out[r0:r0 + 4096] = big_rows(np.arange(r0, min(r0 + 4096, BIG_ROWS)), pool)
    return out


def big_sample_rows():
    """first and last rows, the rows on both sides of 2^31 bytes, and a spread in between"""
    edge = (1 << 31) // (BIG_K * 4)
    return np.unique(np.r_[0, 1, edge - 1, edge, edge + 1, np.linspace(0, BIG_ROWS - 1, 11).astype(np.int64), BIG_ROWS - 1])
