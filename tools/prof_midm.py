"""Mid-M (33..512) options on 4096x4096 4-bit: fused wgmma route, dequantize + dense wgmma (route 3's data flow), the small-M kernel in
chunks of 32 tokens, and cuBLAS on the dequantised matrix -- to decide the router's boundaries."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import ops
from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear

torch.manual_seed(0)
for N, K in ((4096, 4096), (14336, 4096)):
    layer = HQQLinear.from_weights((torch.randn(N, K, device="cuda") * 0.02).half(), None, BaseQuantizeConfig(nbits=4, group_size=64, axis=1),
                                   compute_dtype=torch.float16, device="cuda")
    Wd = layer.dequantize()
    m = layer.meta

    def timed(fn, reps=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps * 1e3

    for M in (16, 32, 48, 64, 96, 128, 256, 512):
        x = torch.randn(M, K, device="cuda").half()
        y = torch.empty(M, N, device="cuda", dtype=torch.float16)
        t_f = timed(lambda: ops.linear_fwd(x, layer.W_q, m["scale"], m["zero"], None, N, K, 64, 4, 1, out=y))
        t_dq = timed(lambda: layer.dequantize())
        t_dense = timed(lambda: ops.dense_gemm(x, Wd, None, out=y))
        t_cublas = timed(lambda: torch.matmul(x, Wd.t(), out=y))

        def chunks():
            for i in range(0, M, 32):
                ops.linear_fwd(x[i:i + 32], layer.W_q, m["scale"], m["zero"], None, N, K, 64, 4, 1, out=y[i:i + 32])

        t_chunk = timed(chunks)
        print(f"N={N} K={K} M={M:4d}: fused {t_f:7.1f} us | dequantize {t_dq:6.1f} + dense wgmma {t_dense:6.1f} = {t_dq + t_dense:6.1f} | small-M x{(M + 31) // 32} {t_chunk:7.1f} | cuBLAS(dequantised) {t_cublas:6.1f}",
              flush=True)
