"""Quantise-only run, layers sharded across ranks (BASELINE configs[3]: Llama-2-70B-shaped, 1 -> 8 GPUs; SURVEY 8e: no collective).

    python tools/quantize_sharded.py [--model 70b|8b] [--blocks N]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/quantize_sharded.py

Every rank generates the fp16 weights of ITS linears on the device (synthetic, seed = layer index), quantises them
(4-bit, gs 64, axis 1, proximal solver) and times only the quantiser with CUDA events; the job time is the max over ranks.
Prints one JSON line: aggregate weights/s and algorithmic GB/s (2.5625 B/weight: fp16 source + packed + fp16 meta)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import harness
from hqq_b200.core.quantize import BaseQuantizeConfig, Quantizer

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="70b", choices=["8b", "70b"])
ap.add_argument("--blocks", type=int, default=0)
args = ap.parse_args()
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=dev)
shape = harness.LLAMA3_70B if args.model == "70b" else harness.LLAMA3_8B
nblocks = args.blocks or shape.n_layers
dims = harness.shard_dims(shape, 1)
layers = [(b, name, dims[name]) for b in range(nblocks) for name in ("q", "k", "v", "o", "gate", "up", "down")]
plan = harness.assign_layers([n * k for _, _, (n, k) in layers], world)
mine = plan[rank]
cfg = BaseQuantizeConfig(nbits=4, group_size=64, axis=1)["weight_quant_params"]
total_ms, weights = 0.0, 0
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for n_done, i in enumerate(mine):
    _, _, (n, k) = layers[i]
    g = torch.Generator(device=dev).manual_seed(i)
    W = (torch.randn(n, k, device=dev, generator=g) * 0.02).half()
    if n_done == 0:  # warm-up (module load, workspace)
        Quantizer.quantize(W, device=dev, compute_dtype=torch.float16, **cfg)
    torch.cuda.synchronize(dev)
    e0.record()
    W_q, meta = Quantizer.quantize(W, device=dev, compute_dtype=torch.float16, **cfg)
    e1.record()
    torch.cuda.synchronize(dev)
    total_ms += e0.elapsed_time(e1)
    weights += n * k
    del W, W_q, meta
t = torch.tensor([total_ms], device=dev)
w = torch.tensor([float(weights)], device=dev)
if world > 1:
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dist.all_reduce(w, op=dist.ReduceOp.SUM)
if rank == 0:
    ms, nw = float(t), float(w)
    print(json.dumps({"metric": "quantize_only_weights_per_s", "value": nw / (ms / 1e3), "unit": "weights/s", "n_gpus": world,
                      "ms_total_max_over_ranks": ms, "weights": nw, "algorithmic_GBps": nw * 2.5625 / (ms / 1e3) / 1e9,
                      "config": {"workload": f"Llama-{'2-70B' if args.model == '70b' else '3-8B'}-shaped quantize-only, {nblocks} blocks x 7 linears, "
                                             "fp16 source, 4-bit gs=64 axis=1, layers sharded by size (no collective)"}}), flush=True)
if world > 1:
    dist.barrier()
    os._exit(0)
