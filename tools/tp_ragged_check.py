"""2+ GPU check of tensor-parallel ragged batches: a tp-way model cut from the full quantised weights (shard_from_full), batch 4 with
ragged=True, runs a packed prefill of prompts of 1, 37, 300 and 120 tokens, 12 greedy steps, a refill of slot 2 and 12 more steps
(fused=True: NCCL all-reduces and the NCCL argmax-key reduction) against the one-GPU model of the same weights.

    torchrun --nproc-per-node 2 tools/tp_ragged_check.py"""
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
refill = torch.randint(0, shape.vocab, (50,), generator=g, device=dev)
res = {}
for tp in (1, world):
    kw = dict(tp=world, rank=rank, process_group=dist.group.WORLD) if tp > 1 else dict(tp=1, rank=0)
    m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=4096, seed=9, fused=True, batch=4, ragged=True, shard_from_full=True, **kw)
    m.capture()
    m.reset_state()
    toks = [m.prefill(prompts, chunk=128).tolist()]
    for i in range(24):
        if i == 12:
            toks.append(m.prefill([None, None, refill, None]).tolist())
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize()
    res[tp] = (toks, m.pos.tolist())
    if rank == 0:
        print(f"tp={tp}", toks, "pos", m.pos.tolist(), flush=True)
if rank == 0:
    a, b = res[1][0], res[world][0]
    agree = [sum(int(x[s] == y[s]) for x, y in zip(a, b)) for s in range(4)]
    ok = all(x[s] == y[s] for x, y in zip(a[:4], b[:4]) for s in range(4)) and min(agree) >= len(a) - 2 and res[1][1] == res[world][1]
    print("RAGGED-TP", "AGREE" if ok else "DISAGREE", agree, "of", len(a), flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0)
