"""Where should the single-matrix forward hand over from the small-M kernel to the wgmma kernel?  GPU time (CUDA graph of 20 calls)
of both for M = 8 ... 32 on Llama-3-8B-sized matrices, 4-bit gs 64: HQQ_B200_SMALL_M_MAX = 32 (small kernel) against = 1 (wgmma)."""
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


SHAPES = ((1024, 4096), (4096, 4096), (14336, 4096), (4096, 14336), (28672, 4096))
if len(sys.argv) > 1 and sys.argv[1] == "70b-tp8":  # per-rank matrices of the Llama-3-70B shape at tp = 8 (bs = 32 leg of configs[4])
    SHAPES = ((1280, 8192), (8192, 1024), (3584, 8192), (7168, 8192), (8192, 3584))
for N, K in SHAPES:
    layer = HQQLinear.from_weights((torch.randn(N, K, device="cuda") * 0.02).half(), None, BaseQuantizeConfig(nbits=4, group_size=64, axis=1),
                                   compute_dtype=torch.float16, device="cuda")
    m = layer.meta
    for M in (1, 4, 8, 9, 16, 17, 24, 32):
        x = torch.randn(M, K, device="cuda").half()
        y = torch.empty(M, N, device="cuda", dtype=torch.float16)
        t = {}
        for cap in (32, 1):
            os.environ["HQQ_B200_SMALL_M_MAX"] = str(cap)
            lib.hqq_b200_reload_env()
            if cap == 1 and M == 1:
                t[cap] = float("nan")
                continue
            t[cap] = graph_us(lambda: ops.linear_fwd(x, layer.W_q, m["scale"], m["zero"], None, N, K, 64, 4, 1, out=y))
        del os.environ["HQQ_B200_SMALL_M_MAX"]
        lib.hqq_b200_reload_env()
        print(f"N={N} K={K} M={M:3d}: small-M kernel {t[32]:6.1f} us | wgmma kernel {t[1]:6.1f} us", flush=True)
