"""GPU: falcon_quantize on the device.  b200_quantize_chunks writes, chunk for chunk, the blocks and histograms of the twin
(tests/quantize_file_twin.py, which tests/test_quantize_file.py holds to ggml_quantize_chunk), for all eleven output types; and
b200_quantize_ggcc writes the reference's own output file (falcon_model_quantize from oracle/_ref) byte for byte."""
import numpy as np
import pytest
import pyoracle as po
import quantize_file_twin as tw
import wquant_cases as wc

pytestmark = pytest.mark.gpu

OUT_TYPES = [po.F16, po.Q4_0, po.Q4_1, po.Q5_0, po.Q5_1, po.Q8_0, po.Q2_K, po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K]
FIELDS = {po.Q4_0: [("d", 0, 2), ("qs", 2, 18)], po.Q4_1: [("d", 0, 2), ("m", 2, 4), ("qs", 4, 20)],
          po.Q5_0: [("d", 0, 2), ("qh", 2, 6), ("qs", 6, 22)], po.Q5_1: [("d", 0, 2), ("m", 2, 4), ("qh", 4, 8), ("qs", 8, 24)],
          po.Q8_0: [("d", 0, 2), ("qs", 2, 34)], po.F16: [("value", 0, 2)],
          po.Q2_K: [("scales", 0, 16), ("qs", 16, 80), ("d", 80, 82), ("dmin", 82, 84)],
          po.Q3_K: [("hmask", 0, 32), ("qs", 32, 96), ("scales", 96, 108), ("d", 108, 110)],
          po.Q4_K: [("d", 0, 2), ("dmin", 2, 4), ("scales", 4, 16), ("qs", 16, 144)],
          po.Q5_K: [("d", 0, 2), ("dmin", 2, 4), ("scales", 4, 16), ("qh", 16, 48), ("qs", 48, 176)],
          po.Q6_K: [("ql", 0, 128), ("qh", 128, 192), ("scales", 192, 208), ("d", 208, 210)]}
CASES = [c for c in wc.cases() if c.x.size <= (1 << 21)]


def _first_difference(t, got, want, chunk):
    bb, be = po.BLOCK_BYTES[t], po.BLOCK_ELEMS[t]
    g, w = got.reshape(-1, bb), want.reshape(-1, bb)
    bad = np.flatnonzero((g != w).any(axis=1))
    if bad.size == 0:
        return None
    i = int(bad[0])
    fields = [f for f, lo, hi in FIELDS[t] if not np.array_equal(g[i, lo:hi], w[i, lo:hi])]
    return "%s: %d of %d blocks differ; first: chunk %d block %d, fields %s" % (
        po.TYPE_NAMES[t], bad.size, g.shape[0], i * be // chunk, i % (chunk // be), ",".join(fields))


def _device(gpu, t, x, chunk):
    x = np.ascontiguousarray(x, np.float32).ravel()
    xd, out = gpu.DevBuf(src=x), gpu.DevBuf(max(po.row_bytes(t, x.size), 16))
    hist = np.zeros(16, np.int64)
    nb = gpu.quantize_chunks(t, xd.ptr, out.ptr, x.size, chunk, hist)
    assert nb == po.row_bytes(t, x.size)
    return out.download(np.uint8, (nb,)), hist


@pytest.mark.parametrize("t", OUT_TYPES, ids=[po.TYPE_NAMES[t] for t in OUT_TYPES])
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_chunks_equal_twin(gpu, case, t):
    x = case.x.ravel()
    be = po.BLOCK_ELEMS[t]
    if x.size % max(be, 256) != 0:
        pytest.skip("shape does not apply")
    for chunk in (16384, x.size, be):
        if t in tw.KQUANTS and chunk % 256:
            continue
        want, wh = tw.quantize_chunks(t, x, chunk)
        got, gh = _device(gpu, t, x, chunk)
        diff = _first_difference(t, got, want, chunk)
        assert diff is None, "%s chunk %d: %s" % (case.name, chunk, diff)
        assert gh.tolist() == wh.tolist(), (case.name, chunk)


def test_f16_specials_equal_reference(gpu):
    """+-Inf, subnormals, values that overflow to Inf, ties, NaNs with payloads: the reference's F16C conversion"""
    bits = [0x7f800000, 0xff800000, 0x00000001, 0x80000001, 0x33800000, 0x387fc000, 0x38800000, 0x477fe000, 0x477ff000,
            0x47800000, 0x7f7fffff, 0x7fc00000, 0xffc00000, 0x7f800001, 0x7fa5a5a5, 0xffb0b000, 0x7fbfffff, 0x3f801000,
            0x3f803000, 0x0, 0x80000000]
    x = np.concatenate([np.array(bits, np.uint32).view(np.float32),
                        np.random.default_rng(3).standard_normal(4096 - len(bits)).astype(np.float32) * 1e3])
    got, _ = _device(gpu, po.F16, x, 16384)
    # ggml_quantize_chunk(F16) is ggml_fp32_to_fp16_row, the x86-64-v3 build's F16C conversion
    hist = np.zeros(16, np.int64)
    nb, w = tw.ref_quantize_chunk(po.F16, x, 0, x.size, hist)
    want = w.view(np.uint16)
    assert np.array_equal(got.view(np.uint16), want), np.flatnonzero(got.view(np.uint16) != want)[:8]
    assert not hist.any()


def test_chunks_return_codes(gpu):
    x = gpu.DevBuf(4096 * 4)
    y = gpu.DevBuf(4096 * 4)
    assert gpu.quantize_chunks(po.F32, x.ptr, y.ptr, 4096, 16384) == 0
    assert gpu.quantize_chunks(po.Q8_1, x.ptr, y.ptr, 4096, 16384) == 0
    assert gpu.quantize_chunks(po.Q4_K, x.ptr, y.ptr, 4096 + 32, 16384) == -1
    assert gpu.quantize_chunks(po.Q4_0, x.ptr, y.ptr, 4096, 16) == -1
    assert gpu.quantize_chunks(po.Q4_0, x.ptr, y.ptr, 4096, 0) == -1
    assert gpu.quantize_chunks(po.Q4_0, x.ptr, y.ptr, -32, 32) == -1
    assert gpu.quantize_chunks(po.Q4_0, x.ptr, y.ptr, 0, 32) == 0
    assert gpu.quantize_chunks(po.Q4_0, x.ptr, y.ptr, 4096, 4096) == 4096 // 32 * 18


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    d = tmp_path_factory.mktemp("qfg")
    return {(m, t): tw.write_model(str(d / ("%s_%d.bin" % (m, t))), hp, t)
            for m, hp in (("A", tw.MODEL_A), ("B", tw.MODEL_B)) for t in (po.F32, po.F16, po.Q8_0, po.Q4_K)}


def _device_equals_reference(gpu, tmp_path, src, ftype, nthread, **kw):
    ref, dev, twin = str(tmp_path / "ref.bin"), str(tmp_path / "dev.bin"), str(tmp_path / "twin.bin")
    assert tw.ref_quantize_file(src, ref, ftype, nthread, **kw) == 0
    rc, rep = gpu.quantize_ggcc(src, dev, ftype, nthread, **kw)
    assert rc == 0
    a, b = np.fromfile(ref, np.uint8), np.fromfile(dev, np.uint8)
    assert a.size == b.size, (a.size, b.size)
    bad = np.flatnonzero(a != b)
    assert bad.size == 0, "first differing byte at %d of %d" % (bad[0], a.size)
    want = tw.quantize_file(src, twin, ftype, nthread, **kw)
    assert (rep.size_org, rep.size_new, rep.n_tensors) == (want["size_org"], want["size_new"], want["n_tensors"])
    assert list(rep.hist) == want["hist"].tolist()
    return dev, rep


@pytest.mark.parametrize("nthread", [1, 4])
@pytest.mark.parametrize("wtype", [po.F32, po.F16])
@pytest.mark.parametrize("ftype", [0, 1, 2, 3, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18])
def test_file_equals_reference(gpu, tmp_path, models, ftype, wtype, nthread):
    _device_equals_reference(gpu, tmp_path, models[("A", wtype)], ftype, nthread)


@pytest.mark.parametrize("ftype", [2, 7, 10, 15, 17])
def test_file_single_chunk_tensors(gpu, tmp_path, models, ftype):
    _device_equals_reference(gpu, tmp_path, models[("B", po.F16)], ftype, 4)


@pytest.mark.parametrize("src_type", [po.Q8_0, po.Q4_K])
@pytest.mark.parametrize("ftype", [2, 9, 10, 14, 17, 18])
def test_file_requantize(gpu, tmp_path, models, src_type, ftype):
    _device_equals_reference(gpu, tmp_path, models[("A", src_type)], ftype, 4, allow_requantize=True)


def test_file_leave_output_tensor(gpu, tmp_path, models):
    _device_equals_reference(gpu, tmp_path, models[("A", po.F16)], 15, 4, quantize_output_tensor=False)


def test_file_refusals_and_errors(gpu, tmp_path, models):
    out = str(tmp_path / "o.bin")
    wide = tw.write_model(str(tmp_path / "w.bin"), dict(n_vocab=13, n_embd=4544, n_head=71, n_head_kv=1, n_layer=1, falcon_type=7),
                          po.F16, shapes={"transformer.word_embeddings.weight": (4544, 13)})
    for src, ftype, kw in ((models[("B", po.F16)], 4, {}), (wide, 15, {}), (models[("B", po.Q8_0)], 15, {})):
        assert tw.ref_quantize_file(src, out, ftype, 4, **kw) == 1
        assert gpu.quantize_ggcc(src, out, ftype, 4, **kw)[0] == 1
    assert gpu.quantize_ggcc(str(tmp_path / "missing.bin"), out, 15, 4)[0] == -1
    trunc = str(tmp_path / "t.bin")
    with open(models[("B", po.F16)], "rb") as f:
        data = f.read()
    with open(trunc, "wb") as f:
        f.write(data[:len(data) - 100])
    assert gpu.quantize_ggcc(trunc, out, 15, 4)[0] == -1


def test_pipeline_spans_staging_buffers_and_repeats(gpu, tmp_path):
    """tensors of at least three staging buffers each, with the next tensor read and the previous one written around them; two runs
    give the same bytes, and the file equals the reference's"""
    hp = dict(n_vocab=6151, n_embd=2048, n_head=32, n_head_kv=2, n_layer=1, falcon_type=40)
    src = tw.write_model(str(tmp_path / "big.bin"), hp, po.F16)
    dev, rep = _device_equals_reference(gpu, tmp_path, src, 15, 4)
    import ggllm_cpp_b200.ggcc as ggcc
    big = [n for n, ne in ggcc.falcon_shapes(hp).items() if len(ne) == 2 and ne[0] * ne[1] * 2 >= 3 * rep.staging_bytes]
    assert len(big) >= 4, (big, rep.staging_bytes)
    again = str(tmp_path / "again.bin")
    assert gpu.quantize_ggcc(src, again, 15, 4)[0] == 0
    assert open(dev, "rb").read() == open(again, "rb").read()


def test_device_file_loads(gpu, tmp_path, models):
    """the device-made Q4_K file loads through b200_falcon_load_ggcc and evaluates like the oracle on the same file"""
    import ggllm_cpp_b200.ggcc as ggcc
    out = str(tmp_path / "q.bin")
    assert gpu.quantize_ggcc(models[("A", po.F16)], out, 15, 4)[0] == 0
    hp, tensors = ggcc.read_ggcc(out)
    f = gpu.Falcon(tw.MODEL_A, n_ctx=32, n_batch=4)
    f.load_ggcc(out)
    o = po.OrcFalcon(tw.MODEL_A, tensors, n_ctx=32)
    toks = np.array([1, 2, 3, 4], np.int32)
    got, want = f.eval(toks, 0), o.eval(toks, 0)
    assert np.abs(got - want).max() <= 2e-2 * float(np.abs(want).max())
    f.free()
