"""CPU checks of falcon_perplexity's exact twin (tests/perplexity_twin.py) against the reference.

- twin(glibc)'s softmax probability equals the reference's own softmax (refh_ppl_prob in oracle/_ref/libfalcon_ppl.so, which compiles
  examples/falcon_perplexity/falcon_perplexity.cpp unchanged) bit for bit, on random rows at V = 65,024 and 512, all-equal rows, a
  dominant logit, spreads where most e[i] are subnormal or 0, a target at the maximum and a target whose e is 0.
- How often twin(glibc) and twin(CR) differ is reported, not failed on: glibc's expf / logf are not correctly rounded, and the device
  (held to twin(CR)) evaluates them correctly rounded.
- The chunk / batch / scored-range loop against hand-written index lists: n_ctx < 1024 (scoring starts at n_ctx / 2), n_ctx not a
  multiple of n_batch (including a final one-token batch), n_tokens not a multiple of n_ctx (the tail is dropped), n_tokens < n_ctx."""
import ctypes as C
import os
import numpy as np
import pytest
import perplexity_twin as pt
import sampler_twin as tw

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libfalcon_ppl.so")
pytestmark = pytest.mark.skipif(not os.path.exists(LIB), reason="oracle/_ref/libfalcon_ppl.so is not built (oracle/perplexity.mk)")


@pytest.fixture(scope="module")
def ref_prob():
    L = C.CDLL(LIB)
    L.refh_ppl_prob.restype, L.refh_ppl_prob.argtypes = C.c_float, [C.c_void_p, C.c_int, C.c_int]

    def f(row, t):
        row = np.ascontiguousarray(row, np.float32)
        return np.float32(L.refh_ppl_prob(row.ctypes.data_as(C.c_void_p), row.size, t))
    return f


@pytest.mark.parametrize("V", [65024, 512])
def test_twin_glibc_equals_reference_softmax(ref_prob, V):
    diff = []
    for name, row, t in pt.case_rows(V):
        got, want = pt.prob(row, t, tw.GLIBC), ref_prob(row, t)
        if got.view(np.uint32) != want.view(np.uint32):
            diff.append((name, float(got), float(want)))
    assert not diff, diff


def test_reference_edge_rows(ref_prob):
    """the cases mean what they say: p = 1/V on equal rows, p = 0 (term +inf) for a target whose e underflows"""
    for V in (65024, 512):
        cases = {name: (row, t) for name, row, t in pt.case_rows(V)}
        assert ref_prob(*cases["equal"]) == np.float32(1.0 / V)
        p0 = ref_prob(*cases["target_e_zero"])
        assert p0 == 0 and pt.term(p0, tw.GLIBC) == np.inf
        row, _ = cases["wide0"]
        e = tw.GLIBC.exp(row - row.max())
        assert np.mean(e < np.finfo(np.float32).tiny) > 0.5           # most terms subnormal or 0


def test_report_glibc_vs_cr():
    """how often the two twins differ (reported): p, and the term -logf(p)"""
    n = dp = dt = 0
    for V in (65024, 512):
        for name, row, t in pt.case_rows(V, seed=11):
            pg, pc = pt.prob(row, t, tw.GLIBC), pt.prob(row, t, tw.CR)
            n += 1
            dp += pg.view(np.uint32) != pc.view(np.uint32)
            dt += pt.term(pg, tw.GLIBC).view(np.uint32) != pt.term(pc, tw.CR).view(np.uint32)
    rng = np.random.default_rng(5)
    p = rng.uniform(1e-6, 1, 20000).astype(np.float32)
    dl = int(np.sum(tw.GLIBC.log(p).view(np.uint32) != tw.CR.log(p).view(np.uint32)))
    print("\nglibc vs correctly rounded: p differs on %d of %d case rows, the term on %d; logf differs on %d of %d probabilities"
          % (dp, n, dt, dl, p.size))


def test_plan_short_context():
    """n_ctx 10 < 1024: scoring starts at n_ctx / 2 = 5, ends before n_ctx - 1; the tail after two chunks is dropped"""
    p = pt.plan(25, 10, 4)
    assert p == [(0, [(0, 4), (4, 4), (8, 2)], [(5, 6), (6, 7), (7, 8), (8, 9)]),
                 (10, [(0, 4), (4, 4), (8, 2)], [(5, 16), (6, 17), (7, 18), (8, 19)])]


def test_plan_one_token_batch():
    """n_ctx 9, n_batch 4: batches of 4, 4 and 1; scored k 4..7"""
    assert pt.plan(9, 9, 4) == [(0, [(0, 4), (4, 4), (8, 1)], [(4, 5), (5, 6), (6, 7), (7, 8)])]


def test_plan_long_context():
    """n_ctx 1100 >= 1024: scoring starts at 512; n_batch 512 leaves a last batch of 76"""
    (start, batches, scored), = pt.plan(1100 + 37, 1100, 512)
    assert start == 0 and batches == [(0, 512), (512, 512), (1024, 76)]
    assert [k for k, _ in scored] == list(range(512, 1099)) and all(ti == k + 1 for k, ti in scored)


def test_plan_too_few_tokens():
    assert pt.plan(63, 64, 16) == []


def test_loop_sums_in_order():
    """nll accumulates in double over all chunks so far; ppl[c] = exp(nll / count)"""
    ppl = pt.accumulate([[np.float32(1.0), np.float32(2.0)], [np.float32(3.0)]])
    assert np.array_equal(ppl, np.exp([1.5, 2.0]))
