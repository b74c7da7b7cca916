"""2+ GPU check of tensor-parallel prompt scoring: a tp-way model cut from the full quantised weights (shard_from_full), batch 4,
ragged=True, scores prompts of 1, 37, 300 and 120 tokens against the one-GPU model of the same weights.  Each rank's (lse, tgt) over
its vocabulary shard meet in one all_gather_into_tensor; every rank must return the same log-probabilities, and they must meet the
fp16 prefill bar (relative L2 2e-3) against tp = 1, fused and fused=False alike.

    torchrun --nproc-per-node 2 tools/tp_score_check.py"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import harness

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
dist.init_process_group("nccl", device_id=dev)
shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
g = torch.Generator(device=dev).manual_seed(5)
prompts = [torch.randint(0, shape.vocab, (n,), generator=g, device=dev) for n in (1, 37, 300, 120)]
ok = True
for fused in (True, False):
    res = {}
    for tp in (1, world):
        kw = dict(tp=world, rank=rank, process_group=dist.group.WORLD) if tp > 1 else dict(tp=1, rank=0)
        m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=1024, seed=9, fused=fused, batch=4, ragged=True,
                                shard_from_full=True, **kw)
        res[tp] = torch.cat(m.score(prompts, chunk=128))
        del m
        torch.cuda.empty_cache()
    gathered = [torch.empty_like(res[world]) for _ in range(world)]
    dist.all_gather(gathered, res[world])
    same = all(torch.equal(x, gathered[0]) for x in gathered)
    rel = float((res[world] - res[1]).norm() / res[1].norm())
    ok &= same and rel <= 2e-3
    if rank == 0:
        print("SCORE-TP", f"fused={fused}", "ranks agree" if same else "RANKS DISAGREE", f"rel L2 vs tp=1 {rel:.2e}", flush=True)
if rank == 0:
    print("SCORE-TP", "PASS" if ok else "FAIL", flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0)
