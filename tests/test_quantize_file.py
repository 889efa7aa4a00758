"""CPU tests: the falcon_quantize twin (tests/quantize_file_twin.py) writes the reference's own output file byte for byte
(falcon_model_quantize from oracle/_ref, through ctypes), refuses where the reference refuses, and its histograms are the
reference's, count for count (ggml_quantize_chunk) and as falcon_quantize prints them.

The weights are i.i.d. random on purpose: the reference starts each Q2_K / Q4_K / Q5_K chunk from codes left on the stack, the twin
(like the device) from zeros, and only data whose sub-blocks repeat can tell the two apart."""
import os
import numpy as np
import pytest
import pyoracle as po
import quantize_file_twin as tw

pytestmark = pytest.mark.skipif(not po.have_ref_falcon(), reason="oracle/_ref is not built")

FTYPES = [0, 1, 2, 3, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18]


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    d = tmp_path_factory.mktemp("qf")
    return {(m, t): tw.write_model(str(d / ("%s_%d.bin" % (m, t))), hp, t)
            for m, hp in (("A", tw.MODEL_A), ("B", tw.MODEL_B)) for t in (po.F32, po.F16, po.Q8_0, po.Q4_K)}


def _same_as_reference(tmp_path, src, ftype, nthread, **kw):
    ref, twin = str(tmp_path / "ref.bin"), str(tmp_path / "twin.bin")
    assert tw.ref_quantize_file(src, ref, ftype, nthread, **kw) == 0
    rep = tw.quantize_file(src, twin, ftype, nthread, **kw)
    a, b = np.fromfile(ref, np.uint8), np.fromfile(twin, np.uint8)
    assert a.size == b.size, (a.size, b.size)
    bad = np.flatnonzero(a != b)
    assert bad.size == 0, "first differing byte at %d of %d" % (bad[0], a.size)
    return rep


@pytest.mark.parametrize("nthread", [1, 4])
@pytest.mark.parametrize("wtype", [po.F32, po.F16])
@pytest.mark.parametrize("ftype", FTYPES)
def test_twin_file_equals_reference(tmp_path, models, ftype, wtype, nthread):
    _same_as_reference(tmp_path, models[("A", wtype)], ftype, nthread)


@pytest.mark.parametrize("ftype", [2, 7, 9, 10, 15, 17, 18])
def test_twin_single_chunk_tensors(tmp_path, models, ftype):
    """embedding and head of one chunk: nthread 4 still makes them one ggml_quantize_chunk call"""
    _same_as_reference(tmp_path, models[("B", po.F16)], ftype, 4)


@pytest.mark.parametrize("src_type", [po.Q8_0, po.Q4_K])
@pytest.mark.parametrize("ftype", [2, 8, 10, 14, 17, 18])
def test_twin_requantize(tmp_path, models, src_type, ftype):
    _same_as_reference(tmp_path, models[("A", src_type)], ftype, 4, allow_requantize=True)


@pytest.mark.parametrize("ftype", [3, 15])
def test_twin_leave_output_tensor(tmp_path, models, ftype):
    _same_as_reference(tmp_path, models[("A", po.F16)], ftype, 4, quantize_output_tensor=False)


def _wide_7b(path):
    """a 7B-width file: only what the reference's loader needs before it meets the first tensor to quantise (it reads 12 special
    tokens, so the vocabulary has at least that many)"""
    hp = dict(n_vocab=13, n_embd=4544, n_head=71, n_head_kv=1, n_layer=1, falcon_type=7)
    return tw.write_model(path, hp, po.F16, shapes={"transformer.word_embeddings.weight": (4544, 13)})


@pytest.mark.parametrize("case", ["ftype4", "width4544", "requantize"])
def test_refusals(tmp_path, models, case):
    out = str(tmp_path / "out.bin")
    src, ftype, kw = {"ftype4": (models[("B", po.F16)], 4, {}),
                      "width4544": (_wide_7b(str(tmp_path / "w.bin")), 15, {}),
                      "requantize": (models[("B", po.Q8_0)], 15, {})}[case]
    assert tw.ref_quantize_file(src, out, ftype, 4, **kw) == 1
    with pytest.raises(tw.Refused):
        tw.quantize_file(src, out, ftype, 4, **kw)
    if case == "width4544":          # a legacy type takes the same tensor
        _same_as_reference(tmp_path, src, 2, 4)


@pytest.mark.parametrize("t", tw.LEGACY)
@pytest.mark.parametrize("chunk", [16384, 32, None])
def test_legacy_hist_equals_ggml_quantize_chunk(t, chunk):
    """the twin's histograms and blocks equal what ggml_quantize_chunk adds and writes, chunk by chunk, q5's shift quirk included"""
    rng = np.random.default_rng(t)
    x = (rng.standard_normal(768 * 61) * rng.choice([0.02, 1.0, 30.0], 768 * 61)).astype(np.float32)
    chunk = chunk or x.size
    want = np.zeros(16, np.int64)
    blocks = []
    for s in range(0, x.size, chunk):
        n = min(chunk, x.size - s)
        nb, y = tw.ref_quantize_chunk(t, x, s, n, want)
        assert nb == po.row_bytes(t, n)
        blocks.append(y)
    got_blocks, got = tw.quantize_chunks(t, x, chunk)
    assert np.array_equal(np.concatenate(blocks), got_blocks)
    assert got.tolist() == want.tolist()
    assert got.sum() == x.size


@pytest.mark.parametrize("ftype", [2, 3, 7, 8, 9])
def test_printed_hists_equal_twin(tmp_path, models, capfd, ftype):
    src = models[("A", po.F16)]
    capfd.readouterr()
    assert tw.ref_quantize_file(src, str(tmp_path / "r.bin"), ftype, 4) == 0
    printed = tw.parse_printed_hists(capfd.readouterr().out)
    rep = tw.quantize_file(src, str(tmp_path / "t.bin"), ftype, 4)
    assert len(printed) == len(rep["per_tensor"])
    for row, (name, h) in zip(printed, rep["per_tensor"].items()):
        n = int(h.sum())
        assert row == [float("%5.3f" % np.float32(np.float32(c) / np.float32(n))) for c in h], name
