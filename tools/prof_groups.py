"""Launch each of the four per-block launch groups of a decode step (q+k+v, o, gate+up, down; Llama-3-8B shapes, 4-bit gs=64)
on cold weights -- the target of the `ncu --set full` capture whose dram bytes fill bench.py's roofline.traffic.

    ncu --set full --clock-control none --import-source on -k regex:linear_decode1 -o prof_groups python tools/prof_groups.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import ops
from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear

groups = [("qkv", 4096, (4096, 1024, 1024)), ("o", 4096, (4096,)), ("gate_up", 4096, (14336, 14336)), ("down", 14336, (4096,))]
torch.manual_seed(0)
cfg = BaseQuantizeConfig(nbits=4, group_size=64, axis=1)
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
for name, K, Ns in groups:
    layers = [HQQLinear.from_weights((torch.randn(N, K, device="cuda") * 0.02).half(), None, cfg, compute_dtype=torch.float16, device="cuda")
              for N in Ns]
    x = torch.randn(1, K, device="cuda").half()
    outs = [torch.empty(1, N, device="cuda", dtype=torch.float16) for N in Ns]
    flush.fill_(1)  # evict the freshly written weights from the 50 MB L2
    torch.cuda.synchronize()
    assert ops.decode_linear_fwd(x, layers, outs, ops.YOP_SILU_MUL_PAIR if name == "gate_up" else 0)  # the MLP launch ships paired
    torch.cuda.synchronize()
    nbytes = sum(N * K // 2 + 2 * (N * K // 64) * 2 for N in Ns) + (Ns[0] if name == "gate_up" else sum(Ns)) * 2 + K * 2
    print(f"{name}: K={K} N={Ns} algorithmic_bytes={nbytes}", flush=True)
