"""CPU tests of the exact-arithmetic attention reference (tests/attn_exact.py) that the GPU attention tests compare against.

  * with fp32 inputs it agrees, within its own bound, with the oracle-built restatement of test_real_geometry_gpu.py
  * the bound is tight enough to catch the defects an attention kernel typically has: a key leaking past the causal limit, a
    visible key dropped at a 128-key tile edge, one key's V row taken from the neighbouring KV head.  Each of these moves at least
    one output element by 10x its bound, so a GPU test that holds a kernel to the bound fails on them.
"""
import numpy as np
import pytest
import attn_exact as ax
from test_real_geometry_gpu import _attention_ref


def _inputs(seed, n_tok, n_past, n_head, n_head_kv):
    rng = np.random.default_rng(seed)
    T = n_past + n_tok
    q = rng.standard_normal((n_tok, n_head, 64)).astype(np.float32)
    K = rng.standard_normal((T, n_head_kv, 64)).astype(np.float32)
    V = rng.standard_normal((T, n_head_kv, 64)).astype(np.float32)
    return q, K, V


@pytest.mark.parametrize("n_head,n_head_kv,n_tok,n_past", [(32, 2, 9, 121), (71, 1, 3, 60), (16, 8, 5, 11), (128, 8, 1, 300)])
def test_reference_agrees_with_oracle_softmax(orc, n_head, n_head_kv, n_tok, n_past):
    """kind "fp32" against _attention_ref (orc.soft_max: ggml's fp16-LUT softmax, fp32 P V): within the bound everywhere, and the
    bound is small (the LUT makes the two differ only where a score sits at an fp16 rounding midpoint)"""
    rng = np.random.default_rng(n_head + n_tok)
    hd, n_ctx = 64, 512
    qkv = rng.standard_normal((n_tok, (n_head + 2 * n_head_kv) * hd)).astype(np.float32)
    kc = rng.standard_normal((n_ctx, n_head_kv, hd)).astype(np.float32)
    vc = rng.standard_normal((n_ctx, n_head_kv, hd)).astype(np.float32)
    want, k_new, v_new = _attention_ref(orc, qkv, kc, vc, n_head, n_head_kv, n_past, n_ctx)
    q = orc.rope_neox(qkv.reshape(n_tok, -1, hd)[:, :n_head], n_past, n_ctx)
    K, V = np.concatenate([kc[:n_past], k_new]), np.concatenate([vc[:n_past], v_new])
    out, bound = ax.reference(q, K, V, n_past, "fp32")
    err = np.abs(out - want)
    assert np.all(err <= bound), float((err / bound).max())
    assert np.median(err) < 1e-6 and np.median(bound) < 5e-3 * np.median(np.abs(want))


def _max_ratio(a, b, bound):
    return float((np.abs(a - b) / bound).max())


@pytest.mark.parametrize("kind", ax.KINDS)
@pytest.mark.parametrize("n_head,n_head_kv,n_tok,n_past", [(32, 2, 64, 1984), (142, 2, 9, 121)])
def test_bound_catches_leaks_drops_and_wrong_heads(kind, n_head, n_head_kv, n_tok, n_past):
    """T = 2048 with G = 16 and T = 130 with G = 71 (standard-normal q, k, v): each mutated reference misses the bound of the true one
    by at least 10x on some element"""
    q, K, V = _inputs(n_tok + n_past, n_tok, n_past, n_head, n_head_kv)
    T = n_past + n_tok
    want, bound = ax.reference(q, K, V, n_past, kind)
    mutants = {"first key past the causal limit": dict(vis_offset=1),
               "first key of the last full 128-key tile dropped": dict(drop_key=(T - 1) // 128 * 128 - 128),
               "last key of a 128-key tile dropped": dict(drop_key=127),
               "one V row from the neighbouring KV head": dict(v_swap_key=n_past - 1)}
    for what, kw in mutants.items():
        got, _ = ax.reference(q, K, V, n_past, kind, **kw)
        r = _max_ratio(got, want, bound)
        assert r >= 10, (kind, what, r)


def test_flat_softmax_is_the_exact_mean():
    """q = 0: every e is exactly 1, the reference output is the mean of the visible V rows and the bound is the accumulation term alone"""
    q, K, V = _inputs(3, 9, 119, 8, 2)
    q[:] = 0
    for kind in ax.KINDS:
        out, bound = ax.reference(q, K, V, 119, kind)
        Vk = ax.f16(V) if kind == "ws" else V.astype(np.float64)
        for t in range(9):
            mean = Vk[:120 + t].mean(0)                                         # [n_head_kv][64]
            assert np.allclose(out[t].reshape(2, 4, 64), mean[:, None, :], rtol=0, atol=1e-6)          # fp32(1 / sum) is the only rounding
        assert bound.max() < 1e-4
