"""Time the fused wgmma dequant-GEMM over the BASELINE sweep (and cuBLAS on the dequantised matrix for reference)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import ops
from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear

shapes = [(4096, 4096), (11008, 4096), (4096, 11008)]
Ms = [int(v) for v in sys.argv[1].split(",")] if len(sys.argv) > 1 else [4096]
bits = [int(v) for v in sys.argv[2].split(",")] if len(sys.argv) > 2 else [4]
torch.manual_seed(0)
for nbits in bits:
    for N, K in shapes:
        layer = HQQLinear.from_weights((torch.randn(N, K, device="cuda") * 0.02).half(), None, BaseQuantizeConfig(nbits=nbits, group_size=64, axis=1),
                                       compute_dtype=torch.float16, device="cuda")
        Wd = layer.dequantize()
        for M in Ms:
            x = torch.randn(M, K, device="cuda").half()
            y = torch.empty(M, N, device="cuda", dtype=torch.float16)
            nb = layer.meta["nbits"]

            fused = ops.linear_route(M, N, K, 64, nb, 1, x.dtype) != 0  # 3-bit has no fused kernel: dequantise kernel + library GEMM

            def run():
                if fused:
                    return ops.linear_fwd(x, layer.W_q, layer.meta["scale"], layer.meta["zero"], None, N, K, 64, nb, 1, out=y)
                with torch.no_grad():
                    return layer(x)

            for fn, name in ((run, "fused" if fused else "fused(dequant+gemm)"), (lambda: torch.matmul(x, Wd.t(), out=y), "cublas(dequantised)")):
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                reps = 10
                e0.record()
                for _ in range(reps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / reps
                print(f"nbits={nbits} N={N} K={K} M={M} {name:22s}: {ms * 1e3:9.1f} us  {2.0 * M * N * K / ms / 1e9:8.1f} TFLOP/s", flush=True)
