"""2+ GPU check of tensor-parallel paged KV caches: a tp-way model cut from the full quantised weights (shard_from_full), batch 4,
ragged=True, kv_pages=64, runs a packed prefill of prompts of 1, 37, 300 and 120 tokens, 12 greedy decode() steps, a fork of slot 2
into slot 1, a refill of slot 3 and 12 more steps, against the one-GPU paged model of the same weights.  Every rank runs the same host
page logic, so the ranks' page tables must agree too.

    torchrun --nproc-per-node 2 tools/tp_paged_check.py"""
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
    m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=4096, seed=9, fused=True, batch=4, ragged=True, kv_pages=64,
                            shard_from_full=True, **kw)
    m.capture()
    m.reset_state()
    toks = [m.prefill(prompts, chunk=128).tolist()]
    for i in range(24):
        if i == 12:
            m.fork(2, 1)
            toks.append(m.prefill([None, None, None, refill]).tolist())
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize()
    table = m.page_table.clone()
    if tp > 1:  # the ranks' tables agree
        tabs = [torch.empty_like(table) for _ in range(world)]
        dist.all_gather(tabs, table)
        assert all(torch.equal(t, table) for t in tabs)
    res[tp] = (toks, m.pos.tolist(), table.tolist())
    if rank == 0:
        print(f"tp={tp}", toks, "pos", m.pos.tolist(), flush=True)
if rank == 0:
    a, b = res[1][0], res[world][0]
    agree = [sum(int(x[s] == y[s]) for x, y in zip(a, b)) for s in range(4)]
    ok = all(x[s] == y[s] for x, y in zip(a[:4], b[:4]) for s in range(4)) and min(agree) >= len(a) - 2 and res[1][1:] == res[world][1:]
    print("PAGED-TP", "AGREE" if ok else "DISAGREE", agree, "of", len(a), flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0)
