"""Micro-benchmark of the decode mat-vec kernel on model shapes (needs an H100).
Rotates through enough distinct weight matrices that every launch reads cold HBM (> 50 MB L2)."""
import sys, os, json
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ggllm_cpp_b200.binding as b
from bench import peaks

def main():
    b.init(0)
    L = b.lib()
    types = [int(t) for t in sys.argv[1].split(",")] if len(sys.argv) > 1 else [12, 2, 11, 14]
    shapes = [(8192, 9216), (8192, 8192), (8192, 32768), (32768, 8192), (8192, 65024)]
    if len(sys.argv) > 2:
        shapes = [tuple(int(v) for v in sh.split("x")) for sh in sys.argv[2].split(",")]
    e0, e1 = L.b200_event_create(), L.b200_event_create()
    for t in types:
        for K, M in shapes:
            blk, bb = {2: (32, 18), 3: (32, 20), 6: (32, 22), 7: (32, 24), 8: (32, 34), 10: (256, 84), 11: (256, 110), 12: (256, 144), 13: (256, 176), 14: (256, 210)}[t]
            nbytes = K // blk * bb * M
            nmat = max(2, int(400e6 // nbytes) + 1)
            Ws = [b.Weight(t, K, M, seed=i + 1) for i in range(nmat)]
            x = np.random.default_rng(0).standard_normal((1, K)).astype(np.float32)
            xd, yd = b.DevBuf(src=x), b.DevBuf(M * 4)
            A = b.ActQ(t, K, 1); A.quantize(xd.ptr)
            for w in Ws: L.b200_mul_mat_vec_q(w.h, A.h, yd.ptr, M, 0, None, None)
            L.b200_synchronize()
            reps = 5
            L.b200_event_record(e0, None)
            for _ in range(reps):
                for w in Ws: L.b200_mul_mat_vec_q(w.h, A.h, yd.ptr, M, 0, None, None)
            L.b200_event_record(e1, None); L.b200_event_synchronize(e1)
            ms = L.b200_event_elapsed_ms(e0, e1) / (reps * nmat)
            print(json.dumps(dict(type=t, K=K, M=M, us=round(ms * 1e3, 2), GBs=round(nbytes / ms / 1e6, 1), frac_of_peak=round(nbytes / ms / 1e6 / peaks()[0], 3))), flush=True)
            for w in Ws: w.free()

if __name__ == "__main__":
    main()
