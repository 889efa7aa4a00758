"""-m gpu: the drop-in boundary.  The UNMODIFIED reference (ggml.c + libfalcon.cpp compiled with -DGGML_USE_CUBLAS into
oracle/_ref/libfalcon_hook.so, ggml_cuda_* symbols left undefined) is loaded on top of libggml_b200.so, so its own
loader (ggml_cuda_transform_tensor, libfalcon.cpp:1251), graph builder and executor hook (ggml_cuda_compute_forward,
ggml.c:15779-15790) drive our kernels.  Logits are compared with the oracle's CPU restatement."""
import os
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model, ggcc

pytestmark = pytest.mark.gpu
HOOK = os.path.join(po.HERE, "_ref", "libfalcon_hook.so")


@pytest.mark.skipif(not os.path.exists(HOOK), reason="oracle/_ref/libfalcon_hook.so not present (built by make -C oracle ref from the reference sources)")
@pytest.mark.parametrize("takeover", [True, False])
@pytest.mark.parametrize("hp,wt,ftype,overrides", [(TINY_40B, po.Q4_K, 15, None), (TINY_7B, po.Q4_0, 2, None),
                                                   (TINY_40B, po.Q4_K, 15, {"lm_head": po.F16})])      # a --leave-output-tensor file
def test_reference_eval_runs_on_our_operator_surface(gpu, tmp_path, hp, wt, ftype, overrides, takeover, monkeypatch):
    """takeover=True: from the second falcon_eval on, the hook recognises the Falcon graph and evaluates it whole on the device-resident
    engine (ggml_surface.cu "whole-graph takeover"); False (B200_NO_TAKEOVER=1): every claimed node goes through the per-node protocol."""
    if not takeover:
        monkeypatch.setenv("B200_NO_TAKEOVER", "1")
    taken0 = gpu.lib().b200_surface_takeover_evals()
    tensors = synth_model(hp, wt, seed=1234, overrides=overrides)
    path = str(tmp_path / "m.ggcc")
    ggcc.write_ggcc(path, hp, tensors, ftype=ftype)
    gpu.lib()                                      # libggml_b200.so is in the global symbol scope (RTLD_GLOBAL)
    ref = po.RefFalcon(path, n_ctx=64, n_batch=16, logits_all=True, hook=True, n_gpu_layers=99)
    o = po.OrcFalcon(hp, tensors, n_ctx=64)
    # (1) batches of <= 8 tokens and decode steps take the hook's integer mat-vec branch: same integers as the CPU, so most evals must
    #     sit at the fp32-reassociation level ("tight", tests/test_falcon_gpu.py), every one inside the loose bound
    short = np.array([11, 100, 101, 102, 103, 104], np.int32)
    got, want = ref.eval(short, 0, n_threads=2), o.eval(short, 0, all_logits=True)
    S = np.abs(want).max()
    assert np.abs(got - want).max() <= 2e-2 * S and np.median(np.abs(got - want)) <= 2e-3 * S
    tight = [bool(np.median(np.abs(got - want)) <= 2e-5 * S)]
    for i in range(4):
        tok = np.array([200 + i], np.int32)
        g, w = ref.eval(tok, 6 + i, n_threads=2), o.eval(tok, 6 + i, all_logits=True)
        assert np.abs(g - w).max() <= 2e-2 * S and np.median(np.abs(g - w)) <= 2e-3 * S
        tight.append(bool(np.median(np.abs(g - w)) <= 2e-5 * S))
    assert sum(tight) * 2 >= len(tight), tight
    # (2) 12 tokens: the N > 8 (wgmma GEMM, fp16 operands) branch of the hook, then decode over the KV cache it wrote.
    #     Tolerance: the GEMM-path bound (max 3e-2 * S, median 5e-3 * S)
    prompt = np.array([11] + list(range(100, 111)), np.int32)
    got, want = ref.eval(prompt, 0, n_threads=2), o.eval(prompt, 0, all_logits=True)
    assert np.abs(got - want).max() <= 3e-2 * S and np.median(np.abs(got - want)) <= 5e-3 * S
    for i in range(3):
        tok = np.array([300 + i], np.int32)
        g, w = ref.eval(tok, 12 + i, n_threads=2), o.eval(tok, 12 + i, all_logits=True)
        assert np.abs(g - w).max() <= 3e-2 * S and np.median(np.abs(g - w)) <= 5e-3 * S
    taken = gpu.lib().b200_surface_takeover_evals() - taken0
    assert taken == (8 if takeover else 0), taken          # every eval after the first ("learning") one ran on the engine
    ref.close()
