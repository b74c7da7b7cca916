"""GPU time (CUDA graph of 20 calls, so no host launch overhead) of the fused wgmma route at mid M against the largest number of
k-slices the schedule may use (HQQ_B200_GEMM_KSPLIT = 1 / 2 / 4 / 8), with the reference's flow (dequantize kernel + cuBLAS) and
cuBLAS alone on the dequantised matrix beside it."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import _lib, ops
from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear

lib = _lib.load()
torch.manual_seed(0)
REP = 20


def graph_us(fn):
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REP):
            fn()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (5 * REP) * 1e3


shapes = ((4096, 4096), (14336, 4096), (4096, 14336)) if len(sys.argv) < 2 else (tuple(int(v) for v in sys.argv[1].split("x")),)
for N, K in shapes:
    layer = HQQLinear.from_weights((torch.randn(N, K, device="cuda") * 0.02).half(), None, BaseQuantizeConfig(nbits=4, group_size=64, axis=1),
                                   compute_dtype=torch.float16, device="cuda")
    Wd = layer.dequantize()
    m = layer.meta
    for M in (33, 64, 128, 256, 384, 512, 768, 1024, 1536, 2048):
        x = torch.randn(M, K, device="cuda").half()
        y = torch.empty(M, N, device="cuda", dtype=torch.float16)
        t = {}
        for cap in (1, 2, 4, 8):
            os.environ["HQQ_B200_GEMM_KSPLIT"] = str(cap)
            lib.hqq_b200_reload_env()
            t[cap] = graph_us(lambda: ops.linear_fwd(x, layer.W_q, m["scale"], m["zero"], None, N, K, 64, 4, 1, out=y))
        del os.environ["HQQ_B200_GEMM_KSPLIT"]
        lib.hqq_b200_reload_env()
        t_ref = graph_us(lambda: torch.matmul(x, layer.dequantize().t(), out=y))
        t_cub = graph_us(lambda: torch.matmul(x, Wd.t(), out=y))
        print(f"N={N} K={K} M={M:5d}: fused, at most 1/2/4/8 k-slices: " + " ".join(f"{t[c]:6.1f}" for c in (1, 2, 4, 8)) +
              f" us | dequantize + cuBLAS {t_ref:6.1f} | cuBLAS alone {t_cub:6.1f}", flush=True)
