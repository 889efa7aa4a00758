"""-m gpu: falcon_perplexity's scoring on the device, held to the exact twin (tests/perplexity_twin.py, correctly rounded expf / logf).

1. b200_token_nll equals twin(CR) bit for bit on the edge rows of perplexity_twin.case_rows at V = 65,024 (strided rows too); a target
   outside [0, V) writes NaN and -1 leaves its slot untouched.
2. b200_falcon_score's terms equal twin(CR) over b200_falcon_eval(all_logits = 1)'s logits for the same batches, bit for bit: batches of
   1 (decode step graph), 5 (mat-vec head) and 40 tokens (GEMM head); Q4_K / Q4_0, f32 and fp16 KV cache, a mixed-type model on the
   generic path, and the 2-layer Falcon-40B-width model with n_vocab 65,024.  A batch with no scored row (no head) leaves the cache as
   an eval does.
3. b200_falcon_perplexity's ppl and terms equal the twin's loop over b200_falcon_eval(all_logits = 1)'s logits bit for bit: two chunks
   plus a dropped tail, n_ctx 64 / 49 / 1100 (scoring from n_ctx / 2 and from 512), short last batches including a one-token one.
4. Against the oracle's falcon_eval restatement: -log p is 2-Lipschitz in the max-norm of the logits, so every device term lies within
   2 max_i |l_dev,i - l_orc,i| (that row's difference) + 1e-5 (1 + term) of twin(CR) over the oracle's logits, and the perplexity
   within the bound those terms imply.
5. Argument checks: bad targets return 3, bad tokens 2, n_ctx above the engine's capacity or below 2 -1, n_tokens < n_ctx 0 chunks."""
import ctypes as C
import numpy as np
import pytest
import pyoracle as po
import perplexity_twin as pt
import sampler_twin as tw
from helpers import TINY_40B, TINY_7B, synth_model

pytestmark = pytest.mark.gpu

MIXED = {"dense_4h_to_h": po.Q6_K, "query_key_value": po.Q5_0, "lm_head": po.Q8_0}
MODELS = {"40b_q4_k": (TINY_40B, po.Q4_K, None), "7b_q4_0": (TINY_7B, po.Q4_0, None), "40b_mixed": (TINY_40B, po.Q4_K, MIXED)}


def bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def batch_targets(rng, toks, V, skip_every=3):
    """next-token targets with every skip_every-th row skipped (-1)"""
    t = rng.integers(0, V, toks.size).astype(np.int32)
    t[::skip_every] = -1
    return t


def test_token_nll_kernel(gpu):
    V = 65024
    cases = pt.case_rows(V, seed=3)
    rows = np.stack([r for _, r, _ in cases])
    targets = np.array([t for _, _, t in cases] + [-1, V, -2, 1 << 30], np.int32)
    rows = np.concatenate([rows, rows[:4]])                            # the last four rows: skipped / out-of-range targets
    want = pt.terms(rows[:len(cases)], targets[:len(cases)], tw.CR)
    for stride in (V, V + 37):
        x = np.zeros((rows.shape[0], stride), np.float32)
        x[:, :V] = rows
        x[:, V:] = 1e30                                                 # padding the kernel must not read
        lg, tg = gpu.DevBuf(src=x), gpu.DevBuf(src=targets)
        out = gpu.DevBuf(src=np.full(targets.size, 7.0, np.float32))
        gpu.token_nll(lg.ptr, V, targets.size, tg.ptr, out.ptr, row_stride=stride)
        got = out.download(np.float32, targets.size)
        n = len(cases)
        assert bits_equal(got[:n], want[:n]), [(c[0], float(g), float(w)) for c, g, w in zip(cases, got, want) if g != w]
        assert got[n] == 7.0 and np.isnan(got[n + 1:]).all(), got[n:]
    assert np.isinf(want[[i for i, c in enumerate(cases) if c[0] == "target_e_zero"]]).all()


_engines = {}


def engine(gpu, key, kv_f16, n_ctx=128, n_batch=64):
    k = (key, kv_f16, n_ctx, n_batch)
    if k not in _engines:
        hp, wt, ov = MODELS[key]
        tensors = synth_model(hp, wt, seed=4321, overrides=ov)
        f = gpu.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch, kv_f16=kv_f16)
        f.set_tensors(tensors)
        _engines[k] = (f, tensors)
    return _engines[k]


def score_vs_eval(f, V, seed):
    """test 2's batches on engine f: -> [(tokens, n_past, targets, device logits, device terms)]"""
    rng = np.random.default_rng(seed)
    out = []
    batches = [(rng.integers(0, V, 40).astype(np.int32), 0), (rng.integers(0, V, 5).astype(np.int32), 40),
               (rng.integers(0, V, 1).astype(np.int32), 45)]
    for toks, n_past in batches:
        tg = batch_targets(rng, toks, V) if toks.size > 1 else rng.integers(0, V, 1).astype(np.int32)
        logits = f.eval(toks, n_past, all_logits=True)
        terms = f.score(toks, n_past, tg)
        want = pt.terms(logits, tg, tw.CR)
        assert bits_equal(terms, want), (toks.size, n_past, terms, want)
        out.append((toks, n_past, tg, logits, terms))
    # a batch with no scored row runs no head, and the cache rows it writes are the eval's
    toks0, _, _, _, _ = out[0]
    assert np.isnan(f.score(toks0, 0, np.full(toks0.size, -1, np.int32))).all()
    toks1, p1, tg1, _, terms1 = out[1]
    assert bits_equal(f.score(toks1, p1, tg1), terms1)
    return out


@pytest.mark.parametrize("key", sorted(MODELS))
@pytest.mark.parametrize("kv_f16", [False, True])
def test_score_equals_twin_over_eval_logits(gpu, key, kv_f16):
    f, _ = engine(gpu, key, kv_f16)
    score_vs_eval(f, f.n_vocab, seed=1000 + 10 * sorted(MODELS).index(key) + int(kv_f16))


def test_score_at_40b_width_full_vocab(gpu):
    """the 2-layer Falcon-40B-width model (n_embd 8192) with the real vocabulary: 65,024-wide rows through both head paths"""
    from test_real_geometry_gpu import GEOM, random_model
    hp = dict(GEOM["40b"], n_vocab=65024)
    f = gpu.Falcon(hp, n_ctx=128, n_batch=64)
    f.set_tensors(random_model(hp, po.Q4_K, seed=77))
    try:
        score_vs_eval(f, hp["n_vocab"], seed=9)
    finally:
        f.free()


@pytest.mark.parametrize("key,kv_f16", [("40b_q4_k", False), ("7b_q4_0", True), ("40b_mixed", False)])
@pytest.mark.parametrize("n_ctx,n_batch", [(64, 24), (49, 24), (1100, 512)])
def test_perplexity_equals_twin_loop(gpu, key, kv_f16, n_ctx, n_batch):
    f, _ = engine(gpu, key, kv_f16, n_ctx=1100, n_batch=n_batch)
    V = f.n_vocab
    toks = np.random.default_rng(n_ctx + n_batch).integers(0, V, 2 * n_ctx + 17).astype(np.int32)
    ppl, nll = f.perplexity(toks, n_ctx)
    want_ppl, want_nll = pt.perplexity(toks, n_ctx, n_batch, lambda t, p0: f.eval(t, p0, n_ctx, all_logits=True), tw.CR)
    assert ppl.size == 2 and nll.size == 2 * (n_ctx - 1 - min(512, n_ctx // 2))
    assert bits_equal(nll, want_nll)
    assert np.array_equal(ppl, want_ppl), (ppl, want_ppl)


def lipschitz_ok(dev_terms, orc_terms, dl):
    """every |term_dev - term_orc| <= 2 max|dl| + 1e-5 (1 + term); -> the bounds"""
    b = 2.0 * dl + 1e-5 * (1.0 + np.abs(orc_terms))
    assert (np.abs(dev_terms.astype(np.float64) - orc_terms) <= b).all(), (dev_terms, orc_terms, b)
    return b


@pytest.mark.parametrize("key", ["40b_q4_k", "7b_q4_0"])
def test_against_oracle(gpu, key):
    f, tensors = engine(gpu, key, False)
    hp = MODELS[key][0]
    o = po.OrcFalcon(hp, tensors, n_ctx=128)
    for toks, n_past, tg, logits, terms in score_vs_eval(f, f.n_vocab, seed=5):
        lo = o.eval(toks, n_past, all_logits=True)
        dl = np.abs(logits.astype(np.float64) - lo).max(axis=1)
        s = tg >= 0
        lipschitz_ok(terms[s], pt.terms(lo, tg, tw.CR)[s].astype(np.float64), dl[s])
    # the perplexity loop: the bound on each term, averaged, bounds log ppl
    n_ctx, n_batch = 64, 64
    toks = np.random.default_rng(8).integers(0, f.n_vocab, 2 * n_ctx).astype(np.int32)
    ppl, nll = f.perplexity(toks, n_ctx)
    dls = []

    def orc_eval(t, p0):
        lo, ld = o.eval(t, p0, n_ctx, all_logits=True), f.eval(t, p0, n_ctx, all_logits=True)
        dls.append(np.abs(ld.astype(np.float64) - lo).max(axis=1))
        return lo
    oppl, onll = pt.perplexity(toks, n_ctx, n_batch, orc_eval, tw.CR)
    dl = np.concatenate(dls)
    first = min(512, n_ctx // 2)
    dl_scored = np.concatenate([dl[c * n_ctx + first:(c + 1) * n_ctx - 1] for c in range(2)])
    b = lipschitz_ok(nll, onll.astype(np.float64), dl_scored)
    for c in range(2):
        n = (c + 1) * (n_ctx - 1 - first)
        B = b[:n].mean()
        assert abs(np.log(ppl[c]) - np.log(oppl[c])) <= B + 1e-12, (ppl[c], oppl[c], B)


def test_argument_checks(gpu):
    f, _ = engine(gpu, "40b_q4_k", False)
    L, V = f.L, f.n_vocab
    toks = np.arange(4, dtype=np.int32)
    out = np.zeros(4, np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)                          # noqa: E731
    for bad in (V, -2, 1 << 30):
        tg = np.array([1, bad, -1, 2], np.int32)
        assert L.b200_falcon_score(f.h, p(toks), 4, 0, 0, p(tg), p(out)) == 3
    assert L.b200_falcon_score(f.h, p(toks), 4, 0, 0, None, p(out)) == 3
    tg = np.array([1, 2, -1, 3], np.int32)
    assert L.b200_falcon_score(f.h, p(np.array([0, V, 1, 2], np.int32)), 4, 0, 0, p(tg), p(out)) == 2
    assert L.b200_falcon_score(f.h, p(toks), 4, 126, 0, p(tg), p(out)) == 1
    long_toks = np.zeros(1000, np.int32)
    ppl, nll = np.zeros(8), np.zeros(8000, np.float32)
    assert L.b200_falcon_perplexity(f.h, p(long_toks), 1000, 129, p(ppl), p(nll)) == -1          # above the engine's n_ctx (128)
    assert L.b200_falcon_perplexity(f.h, p(long_toks), 1000, 1, p(ppl), p(nll)) == -1
    bad = long_toks.copy()
    bad[500] = V
    assert L.b200_falcon_perplexity(f.h, p(bad), 1000, 64, p(ppl), p(nll)) == -1
    assert L.b200_falcon_perplexity(f.h, p(long_toks), 63, 64, p(ppl), p(nll)) == 0
    ppl, nll = f.perplexity(long_toks[:63], 64)
    assert ppl.size == 0 and nll.size == 0
