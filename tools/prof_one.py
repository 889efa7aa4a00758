import sys, os
import numpy as np
sys.path.insert(0, "/root/repo")
import ggllm_cpp_b200.binding as b
b.init(0); L = b.lib()
K, M = int(sys.argv[1]), int(sys.argv[2])
Ws = [b.Weight(12, K, M, seed=i + 1) for i in range(4)]
x = b.DevBuf(src=np.random.default_rng(0).standard_normal(K).astype(np.float32))
yd = b.DevBuf(M * 4)
A = b.ActQ(12, K, 1); A.quantize(x.ptr)
for r in range(3):
    for w in Ws:
        L.b200_mul_mat_vec_q(w.h, A.h, yd.ptr, M, 0, None, None)
L.b200_synchronize()
