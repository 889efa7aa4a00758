"""The fp16-cache twin of the oracle (tests/kv16_twin.py): with an f32 cache it is orc_falcon_eval bit for bit, and with an fp16 cache
every row it stores is fp16-representable and layer 0's rows are f16 of the f32 run's (before any attention output can differ)."""
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model
from kv16_twin import Kv16Twin

PROMPT = np.array([11, 100, 101, 102, 103, 104, 105], np.int32)


def _run(m, n_decode=3):
    out = [m.eval(PROMPT, 0, all_logits=True)]
    for s in range(n_decode):
        out.append(m.eval(np.array([200 + 3 * s], np.int32), PROMPT.size + s))
    return out


@pytest.mark.parametrize("hp,wt", [(TINY_40B, po.Q4_K), (TINY_7B, po.Q4_0)])
def test_twin_with_f32_cache_is_the_oracle_bit_for_bit(orc, hp, wt):
    tensors = synth_model(hp, wt, seed=1234)
    ref = po.OrcFalcon(hp, tensors, n_ctx=64)
    twin = Kv16Twin(orc, hp, tensors, 64, kv_f16=False)
    for a, b in zip(_run(twin), _run(ref)):
        assert np.array_equal(a, b)
    assert np.array_equal(twin.k, ref.k) and np.array_equal(twin.v, ref.v)


@pytest.mark.parametrize("hp,wt", [(TINY_40B, po.Q4_K), (TINY_7B, po.Q4_0)])
def test_twin_fp16_cache_holds_rounded_rows(orc, hp, wt):
    tensors = synth_model(hp, wt, seed=1234)
    t16, t32 = Kv16Twin(orc, hp, tensors, 64, kv_f16=True), Kv16Twin(orc, hp, tensors, 64, kv_f16=False)
    out16, out32 = _run(t16), _run(t32)
    n = PROMPT.size + 3
    for a in (t16.k[:, :n], t16.v[:, :n]):                    # every value the fp16 cache holds is fp16-representable
        assert np.array_equal(a, a.astype(np.float16).astype(np.float32))
    assert not np.array_equal(t32.k[:, :n], t32.k[:, :n].astype(np.float16).astype(np.float32))     # the f32 cache's are not
    assert np.array_equal(t16.k[0, :n], t32.k[0, :n].astype(np.float16).astype(np.float32))
    assert np.array_equal(t16.v[0, :n], t32.v[0, :n].astype(np.float16).astype(np.float32))
    assert not t16.k[:, n:].any() and not t16.v[:, n:].any()
    for i, (a, b) in enumerate(zip(out16, out32)):
        assert np.isfinite(a).all()
        print("step %d: fp16-cache logits vs f32-cache logits max |diff| %.3g (scale %.3g)" % (i, float(np.abs(a - b).max()), float(np.abs(b).max())))
