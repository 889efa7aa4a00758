"""Micro-benchmark of the prompt GEMM (wgmma) on Falcon-40B shapes, N = 512 tokens (needs an H100)."""
import sys, os, json
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ggllm_cpp_b200.binding as b
from bench import peaks

def main():
    b.init(0)
    L = b.lib()
    t = int(sys.argv[1]) if len(sys.argv) > 1 else 12
    N = int(sys.argv[2]) if len(sys.argv) > 2 else 512
    shapes = [(8192, 9216), (8192, 8192), (8192, 32768), (32768, 8192)]
    if len(sys.argv) > 3:
        shapes = [tuple(int(v) for v in sh.split("x")) for sh in sys.argv[3].split(",")]
    e0, e1 = L.b200_event_create(), L.b200_event_create()
    for K, M in shapes:
        W = b.Weight(t, K, M, seed=1)
        xh = (np.random.default_rng(0).standard_normal((N, K))).astype(np.float16)
        xd, yd = b.DevBuf(src=xh), b.DevBuf(N * M * 4)
        for _ in range(2): L.b200_mul_mat_f16(W.h, xd.ptr, K, N, yd.ptr, M, 0, 1)
        L.b200_synchronize()
        reps = 5
        L.b200_event_record(e0, None)
        for _ in range(reps): L.b200_mul_mat_f16(W.h, xd.ptr, K, N, yd.ptr, M, 0, 1)
        L.b200_event_record(e1, None); L.b200_event_synchronize(e1)
        ms = L.b200_event_elapsed_ms(e0, e1) / reps
        fl = 2.0 * K * M * N
        print(json.dumps(dict(type=t, K=K, M=M, N=N, us=round(ms * 1e3, 1), TFLOPs=round(fl / ms / 1e9, 1), frac_of_peak=round(fl / ms / 1e9 / peaks()[1], 3))), flush=True)
        W.free()

if __name__ == "__main__":
    main()
