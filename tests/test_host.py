"""CPU tests of the host-side logic: GGCC reader/writer, layer-range partition, and the 2-rank pipeline hand-off
(gloo, world_size 2) with the oracle standing in for the device stages."""
import os
import sys
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model, ggcc


def test_ggcc_roundtrip(tmp_path):
    hp = dict(TINY_7B)
    tensors = synth_model(hp, po.Q4_0, seed=1)
    p = str(tmp_path / "a.ggcc")
    ggcc.write_ggcc(p, hp, tensors, ftype=2)
    hp2, t2 = ggcc.read_ggcc(p)
    assert {k: hp2[k] for k in hp} == hp and hp2["ftype"] == 2
    assert list(t2) == list(tensors)
    for k in tensors:
        assert t2[k][0] == tensors[k][0] and tuple(t2[k][1]) == tuple(tensors[k][1])
        assert np.array_equal(np.asarray(t2[k][2]), np.ascontiguousarray(tensors[k][2]).view(np.uint8).reshape(-1))
        assert (t2[k][2].ctypes.data - t2[k][2].base.ctypes.data if hasattr(t2[k][2], "base") and t2[k][2].base is not None else 0) % 32 == 0


def test_ggcc_shapes_are_the_loaders():
    s = ggcc.falcon_shapes(dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=60, falcon_type=40))
    assert s["transformer.h.59.self_attention.query_key_value.weight"] == (8192, 9216)
    assert s["transformer.h.0.mlp.dense_4h_to_h.weight"] == (32768, 8192)
    n = sum(int(np.prod(v)) for k, v in s.items() if len(v) == 2 and "word_embeddings" not in k)
    assert n == 41301311488                       # W_elems(40B) of SURVEY.md section 8a
    assert ggcc.tensor_nbytes(12, (8192, 9216)) == 8192 * 9216 // 256 * 144


def test_layer_ranges_cover_the_model():
    from ggllm_cpp_b200.binding import layer_range
    for L in (60, 80, 32, 7):
        for world in (1, 2, 4, 8):
            r = [layer_range(L, k, world) for k in range(world)]
            assert r[0][0] == 0 and r[-1][1] == L
            assert all(r[i][1] == r[i + 1][0] for i in range(world - 1))
            sizes = [b - a for a, b in r]
            assert max(sizes) - min(sizes) <= 1


def _pipeline_worker(rank, world, port, q):
    import torch.distributed as dist
    import torch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ggllm_cpp_b200.binding import layer_range
    hp = dict(TINY_40B, n_layer=5)
    tensors = synth_model(hp, po.Q4_K, seed=8)
    lf, ll = layer_range(hp["n_layer"], rank, world)
    stage = po.OrcFalcon(hp, tensors, n_ctx=32)
    out = []
    for toks, n_past in ((np.array([11, 40, 41], np.int32), 0), (np.array([42], np.int32), 3)):
        resid = None
        if rank > 0:
            buf = torch.zeros(len(toks), hp["n_embd"])
            dist.recv(buf, src=rank - 1)                       # one message per boundary per eval
            resid = buf.numpy()
        r = stage.eval_range(toks, n_past, lf, ll, resid_in=resid, all_logits=True)
        if rank < world - 1:
            dist.send(torch.from_numpy(r), dst=rank + 1)
        else:
            out.append(r)
    if rank == world - 1:
        q.put(out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_pipeline_gloo():
    """world_size 2: rank r owns layers layer_range(L, r, 2), the residual stream crosses the boundary once per eval;
    the last rank's logits equal the single-process evaluation bit for bit."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_pipeline_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    hp = dict(TINY_40B, n_layer=5)
    whole = po.OrcFalcon(hp, synth_model(hp, po.Q4_K, seed=8), n_ctx=32)
    assert np.array_equal(got[0], whole.eval(np.array([11, 40, 41], np.int32), 0, all_logits=True))
    assert np.array_equal(got[1], whole.eval(np.array([42], np.int32), 3, all_logits=True))


def test_bench_stage_ranges_and_byte_counts():
    """bench.py's host logic (no GPU): layer ranges balanced by bytes cover the model contiguously with the last rank relieved by the
    lm_head it also streams; the byte counts are BASELINE.md's"""
    import bench
    assert bench.weight_elems(bench.MODELS["falcon40b"]) * bench.BYTES_PER_WEIGHT[bench.Q4_K] == 23231987712
    assert bench.weight_elems(bench.MODELS["falcon7b"]) * bench.BYTES_PER_WEIGHT[bench.Q4_0] == 3893299200
    assert bench.weight_elems(bench.MODELS["falcon40b"]) * bench.BYTES_PER_WEIGHT[bench.Q3_K] == 17746657280
    assert abs(bench.weight_elems(bench.MODELS["falcon180b"]) * bench.BYTES_PER_WEIGHT[bench.Q4_K] - 100.44e9) < 0.01e9
    assert bench.kv_bytes(bench.MODELS["falcon180b"], 8192) == 80 * 2 * 8192 * 8 * 64 * 4
    for name, hp in bench.MODELS.items():
        per_layer = hp["n_embd"] * ((hp["n_head"] + 2 * hp["n_head_kv"]) * 64 + 9 * hp["n_embd"])
        head = hp["n_embd"] * hp["n_vocab"]
        for world in (1, 2, 4, 8):
            r = bench.stage_ranges(hp, world)
            assert r[0][0] == 0 and r[-1][1] == hp["n_layer"] and all(r[i][1] == r[i + 1][0] for i in range(world - 1))
            loads = [(b - a) * per_layer + (head if i == world - 1 else 0) for i, (a, b) in enumerate(r)]
            assert max(loads) - min(loads) <= per_layer + 1, (name, world, r)       # balanced to within one layer's bytes
            assert all(b > a for a, b in r)


def test_bench_line_contract(monkeypatch, capsys):
    """the JSON line bench.py prints carries every key the driver reads: bench.main() run with the GPU legs replaced by canned
    measurements (the contract lives in main's assembly code, which is what this exercises)"""
    import json
    import bench

    class FakeCx:
        rank, world, local_rank, dist = 0, 1, 0, None
        def make_model(self, *a, **k):
            class M:
                def free(self): pass
            return M()
    canned = {"tok_s": 208.0, "ms_per_step": 4.8, "e2e_tok_s": 205.0, "e2e_ms_per_step": 4.88, "wall_ms_per_step": 4.81, "gpu_launches": 10880,
              "weight_bytes": 23231987712.0, "step_bytes": 23239000000.0, "n_past": [9, 29], "step_achieved_GBs": 4833.0, "step_frac": 0.734,
              "roofline_tok_s": 283.4, "_probe": (12.7, 723, 69696000000)}
    monkeypatch.setattr(bench, "Ctx", FakeCx)
    monkeypatch.setattr(bench, "decode_leg", lambda *a, **k: dict(canned))
    monkeypatch.setattr(bench, "prompt_leg", lambda *a, **k: {"tok_s": 11000.0, "seconds": 0.186, "roofline": {"bound": "tensor", "frac": 0.64}})
    monkeypatch.setattr(bench, "matvec_leg", lambda *a, **k: {"gpu": {"us_per_call": 4.2}})
    monkeypatch.setattr(bench, "FullModelFile", lambda *a, **k: type("F", (), {"close": lambda self: None})())
    monkeypatch.setattr(bench, "dropin_decode", lambda *a, **k: {"value": 93.0, "unit": "tok/s"})
    monkeypatch.setattr(bench, "reference_cpu_decode", lambda *a, **k: {"value": 2.7, "unit": "tok/s", "cores": 16, "kind": "reference", "sample": "canned", "extrapolated": False})
    monkeypatch.setattr(bench.ClockSampler, "__init__", lambda self, dev: None)
    monkeypatch.setattr(bench.ClockSampler, "stop", lambda self: {"sm_mhz": 1965.0, "sm_max_mhz": 1965.0, "reasons": []})
    monkeypatch.setattr(sys, "argv", ["bench.py", "--gpus", "1", "--steps", "20", "--warmup", "5"])
    bench.main()
    d = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline", "prompt", "configs", "e2e_dropin"):
        assert k in d, k
    assert d["metric"] == "falcon40b_q4_k_decode_tokens_per_s" and d["steps"] == 20 and d["warmup"] == 5 and d["n_gpus"] == 1
    assert d["config"]["workload"] and "model" not in d["config"]
    assert set(("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step")) <= set(d["e2e"])
    assert set(("bound", "achieved", "peak", "unit", "frac", "traffic")) <= set(d["roofline"])
    assert abs(d["roofline"]["frac"] - d["roofline"]["achieved"] / d["roofline"]["peak"]) < 1e-9
    assert set(("value", "unit", "cores", "kind", "sample")) <= set(d["cpu_baseline"])
    assert d["higher_is_better"] is True and d["vs_baseline"] is None and d["value"] == 208.0 and d["e2e"]["value"] == 205.0
    assert set(d["configs"]) == {"cfg1", "cfg2", "cfg4", "cfg5"}


def test_fp16_split_products_reach_fp32_dot_accuracy():
    """The arithmetic behind the tensor-core decode attention (attention_long.cu): an fp32 operand is split into fp16 terms hi = f16(x),
    lo = f16(x - hi); products of fp16 pairs are exact in the fp32 accumulator, and hi*hi + hi*lo + lo*hi differs from the exact product by
    the dropped lo*lo term (~2^-22).  Emulated here in numpy: a 64-term dot product through the three-term split is as close to the fp64
    result as a plain fp32 dot product is for query / key magnitudes of 0.3 .. 100; below 0.125 the lo term is an fp16 subnormal and the
    representation error becomes ABSOLUTE, <= 2^-25 per element -- for a score that feeds exp(s - max) that is as good.  The softmax
    weights e = f16(exp(f16(x))) are fp16 values already, so that operand of the second product needs no split."""
    rng = np.random.default_rng(5)
    for mag in (1e-3, 1e-2, 0.3, 1.0, 30.0, 100.0):
        q = (mag * rng.standard_normal((4096, 64))).astype(np.float32)
        k = (mag * rng.standard_normal((4096, 64))).astype(np.float32)
        def split(x):
            hi = x.astype(np.float16)
            lo = (x - hi.astype(np.float32)).astype(np.float16)
            return hi.astype(np.float32), lo.astype(np.float32)
        qh, ql = split(q); kh, kl = split(k)
        # every product of two fp16 values has <= 22 significant bits: exact in fp32; the accumulation is fp32 like the mma's
        terms = np.concatenate([qh * kh, qh * kl, ql * kh], axis=1)
        got = terms.sum(axis=1, dtype=np.float32)
        exact = (q.astype(np.float64) * k.astype(np.float64)).sum(axis=1)
        plain = (q * k).sum(axis=1, dtype=np.float32)
        scale = (np.abs(q.astype(np.float64)) * np.abs(k.astype(np.float64))).sum(axis=1)
        if mag < 0.125:
            bound = 64 * 2.0 ** -24 * max(float(np.abs(q).max()), float(np.abs(k).max()))      # 64 terms x (2^-25 |k| + 2^-25 |q|)
            assert np.abs(got - exact).max() <= bound, (mag, float(np.abs(got - exact).max()), bound)
            continue
        err_split, err_plain = np.abs(got - exact) / scale, np.abs(plain - exact) / scale
        assert err_split.max() <= 4e-7, (mag, float(err_split.max()))                   # 64 terms x 2^-24 rounding + 2^-22 dropped term, with margin
        assert np.median(err_split) <= 4 * np.median(err_plain) + 1e-9, (mag, float(np.median(err_split)), float(np.median(err_plain)))
    e = np.exp(rng.uniform(-12, 0, 10000).astype(np.float16).astype(np.float32)).astype(np.float16)
    assert np.array_equal(e.astype(np.float32).astype(np.float16), e)                    # e is representable: the A operand of E V is exact


def test_launch_list_tool_pivots_an_ncu_csv(tmp_path):
    """tools/launch_list.py (pivots an Nsight Compute launch list): one row per launch, the last COMPLETE
    decode step only, DRAM bytes per mat-vec launch"""
    import subprocess, csv as _csv, json
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = ["ID", "Process ID", "Process Name", "Host Name", "Kernel Name", "Context", "Stream", "Block Size", "Grid Size", "Device", "CC",
           "Section Name", "Metric Name", "Metric Unit", "Metric Value"]
    rows, lid = [hdr], 0
    def launch(name, ns, rd):
        nonlocal lid
        for metric, unit, val in (("gpu__time_duration.sum", "us", ns / 1e3), ("dram__bytes_read.sum", "Mbyte", rd / 1e6), ("dram__bytes_write.sum", "byte", 0)):
            rows.append([str(lid), "1", "python", "box", name, "1", "14", "(256, 1, 1)", "(296, 1, 1)", "0", "10.0", "Command line profiler metrics", metric, unit, "%.6f" % val])
        lid += 1
    for step in range(3):                                   # the third step is cut short by the capture limit
        launch("dequant_rows_kernel(WPlanes, const int *, int, float *, long)", 5000, 1e4)
        for i in range(4 if step < 2 else 2):
            launch("void mmv_fast_kernel<12, 256, 1, 8>(WPlanes, ActQ, float *, long, Epi)", 20000, 80e6)
        launch("attn_dec_scores_kernel(AttnDecArgs)", 6000, 1e5)
    raw, out, tr = tmp_path / "raw.csv", tmp_path / "out.csv", tmp_path / "traffic.json"
    with open(raw, "w", newline="") as f:
        f.write("==PROF== Connected to process 1\n")
        _csv.writer(f, quoting=_csv.QUOTE_ALL).writerows(rows)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "launch_list.py"), str(raw), str(out), "--traffic", str(tr)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    body = [l for l in open(out).read().splitlines()[2:] if l]
    assert len(body) == 6                                    # the second (last complete) step: gather + 4 mat-vecs + scores
    t = json.load(open(tr))
    assert t["matvec_launches_per_step"] == 4 and abs(t["dram_bytes_per_matvec_launch"] - 80e6) < 1.0
    assert "mmv_fast_kernel" in r.stdout and "87.9 %" in r.stdout          # 80 of 91 us
