"""Time per b200_sampler_sample call at n_vocab 65,024 for each whole-chain case (tests/sampling_chain_cases.py) and for falcon_main's
default chain, from CUDA events recorded around each call: the sampling kernel plus the id's 4-byte D2H copy (a few microseconds).

    python tools/sampler_bench.py [--calls 300] [--warmup 30]

The "default" case uses only the default-chain API (b200_sampling_params), so the same script measures a build without the chain
API; the other cases are skipped there.  Prints one JSON line per case, after the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402
import ggllm_cpp_b200.binding as b  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def time_sampler(s, rows, calls, warmup):
    L = b.lib()
    e0, e1 = L.b200_event_create(), L.b200_event_create()
    for i in range(warmup):
        s.sample(rows[i % len(rows)].ptr, 65024)
    total = 0.0
    for i in range(calls):
        L.b200_event_record(e0, None)
        s.sample(rows[i % len(rows)].ptr, 65024)
        L.b200_event_record(e1, None)
        L.b200_event_synchronize(e1)
        total += L.b200_event_elapsed_ms(e0, e1)
    L.b200_event_destroy(e0); L.b200_event_destroy(e1)
    return 1000.0 * total / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    a = ap.parse_args()
    b.init(0)
    print(json.dumps({"card": card()}))
    rng = np.random.default_rng(1)
    rows = []
    for _ in range(8):
        r = (rng.standard_normal(65024) * 3.0).astype(np.float32)
        r[rng.integers(0, 65024, size=5)] += 6.0
        rows.append(b.DevBuf(src=r))
    hist = [int(t) for t in rng.integers(0, 65024, size=100)]
    s = b.Sampler(b.SamplingParams(top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, repeat_last_n=64, seed=1), hist)
    print(json.dumps({"case": "default", "us_per_call": round(time_sampler(s, rows, a.calls, a.warmup), 2)}))
    s.free()
    if not hasattr(b, "SamplingChain"):
        return
    import sampling_chain_cases as sc
    keys = ("top_k", "top_p", "tfs_z", "typical_p", "temp", "repeat_penalty", "frequency_penalty", "presence_penalty", "repeat_last_n",
            "mirostat", "mirostat_tau", "mirostat_eta", "logit_bias")
    for name in sorted(sc.CASES):
        c = sc.CASES[name]
        s = b.Sampler(b.SamplingChain(seed=1, **{k: c[k] for k in keys}), hist)
        print(json.dumps({"case": name, "us_per_call": round(time_sampler(s, rows, a.calls, a.warmup), 2)}))
        s.free()


if __name__ == "__main__":
    main()
