"""CPU: the activation-quantisation edge rows (tests/actq_edges.py) test what they claim, the oracle's quantisers agree with the
reference's compiled ones on every edge row, and the GPU file's parametrisation feeds every edge family to every producer."""
import numpy as np
import pytest
import pyoracle as po
import actq_edges as ae


def _all_block_sets():
    for at in ae.ATYPES:
        yield at, None
        if at == po.Q8_K:
            yield at, 64                                  # the attention hand-over's 64-value head templates


@pytest.mark.parametrize("at,period", list(_all_block_sets()))
def test_every_premise_holds(at, period):
    blocks = ae.edge_blocks(at, period)                  # building asserts each premise; check again and check completeness
    for fam, label, b in blocks:
        ae.premise(at, fam, label, b, period)
    assert {f for f, _, _ in blocks} == set(ae.FAMILIES[at])
    labels = [l for f, l, _ in blocks if f == "E1"]
    pairs = ae.E1_PAIRS[256 if at == po.Q8_K else 32]
    for (i, j), _ in pairs:
        if j < (period or ae.BLK[at]):
            for order in ("+-", "-+"):
                assert any(l.startswith("E1 %d/%d %s" % (i, j, order)) for l in labels), (i, j, order)
    e3 = [l for f, l, _ in blocks if f == "E3"]
    assert any("gelu" in l for l in e3) and any("wide" in l for l in e3) and any("7-bit" in l for l in e3)
    if at == po.Q8_K:                                    # every xor distance of the 256-block reduction
        assert {int(l.split()[1].split("/")[0]) // 8 ^ int(l.split()[1].split("/")[1]) // 8 for l in labels} >= (
            {0, 1, 2, 4} if period == 64 else {0, 1, 2, 4, 8, 16})
    else:
        assert {int(l.split()[1].split("/")[0]) // 8 ^ int(l.split()[1].split("/")[1]) // 8 for l in labels} >= {0, 1, 2}


def test_rows_keep_the_blocks():
    for at in ae.ATYPES:
        rows, labels = ae.edge_rows(at, 4096, min_rows=2)
        assert rows.shape[0] >= 2 and rows.dtype == np.float32
        for r in range(rows.shape[0]):
            for i, l in enumerate(labels[r]):
                if l != "fill":
                    ae.premise(at, ae.family_of(l), l, rows[r, i * ae.BLK[at]:(i + 1) * ae.BLK[at]])


def test_gelu_rows_bring_half_way_products():
    """fp16-grid GELU outputs contain half-way products: a quantiser rounding half away from zero would flip codes on real data"""
    for at in ae.ATYPES:
        g = [b for f, l, b in ae.edge_blocks(at) if l == "E3 gelu"]
        assert len(g) == 4 and all(ae.halfway(at, b).any() for b in g)


@pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref (the compiled reference) is not built")
@pytest.mark.parametrize("wt", [po.Q4_0, po.Q4_1, po.Q4_K])
def test_oracle_quantiser_is_the_reference_on_edge_rows(wt):
    """po.orc().quantize_act == the reference's quantize_row_q_dot (AVX2 quantize_row_q8_0 / q8_1, exported quantize_row_q8_K),
    byte for byte, on every edge row the GPU tests use"""
    import test_actq_edges_gpu as G
    at = po.VEC_DOT_TYPE[wt]
    sets = [ae.edge_rows(at, 4096)[0]]
    if at == po.Q8_K:
        sets.append(ae.edge_rows(at, 4096, period=64)[0])
    if wt in G.CHAIN:
        sets.append(G.chain_rows(wt)[0])
    for x in sets:
        a, b = po.orc().quantize_act(wt, x), po.ref().quantize_act(wt, x)
        assert np.array_equal(a, b), int((a != b).sum())


# the producers of the activation codes (and the fp16 GEMM operand) and the activation types each one supports
PRODUCERS = {"standalone": ae.ATYPES, "ln_cluster": ae.ATYPES, "ln_reg1": ae.ATYPES, "ln_reg2": ae.ATYPES, "ln_smem": ae.ATYPES,
             "attn split": ae.ATYPES, "attn long": ae.ATYPES, "chain": (po.Q8_K, po.Q8_0),
             "plane standalone": ae.ATYPES, "plane ln_reg1": ae.ATYPES, "plane ln_reg2": ae.ATYPES, "plane ln_smem": ae.ATYPES}


def test_parametrisation_reaches_every_producer_and_family():
    """every supported (producer, activation type) pair is run by tests/test_actq_edges_gpu.py on every edge family of that type"""
    import test_actq_edges_gpu as G
    got = G.reached()

    def need(p, at):                                     # the long-context attention kernel takes V rows within fp16's range only
        return set(ae.FAMILIES[at]) - ({"E6"} if p == "attn long" else set())
    missing = [(p, po.TYPE_NAMES[at], sorted(need(p, at) - got.get((p, at), set())))
               for p, ats in PRODUCERS.items() for at in ats if need(p, at) - got.get((p, at), set())]
    assert not missing, missing
    assert {k[0] for k in got} == set(PRODUCERS)
    # the cases behind the keys: each LayerNorm kernel and both attention tiers with every type
    assert set(G.LN_KERNEL.values()) == {"ln_cluster", "ln_reg1", "ln_reg2", "ln_smem"}
    assert {po.VEC_DOT_TYPE[wt] for _, _, wt in G.ATTN} == set(ae.ATYPES)
    assert any(G_ % 4 == 0 for G_, _, wt in G.ATTN if wt == po.Q4_K)            # Q8_K folds into the attention only when G % 4 == 0
