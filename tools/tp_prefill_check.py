"""2+ GPU check of the tensor-parallel prompt prefill: a tp-way model cut from the full quantised weights (shard_from_full) runs
prefill + greedy decode (fused=5, peer-memory exchange in the decode step) against the one-GPU model of the same weights."""
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
prompt = torch.randint(0, shape.vocab, (1, 300), generator=torch.Generator(device=dev).manual_seed(5), device=dev)
res = {}
for tp in (1, world):
    # both models draw the full matrices from the shared generator (shard_from_full): the tp-way model holds shards of exactly the
    # one-GPU model's quantised weights
    kw = dict(tp=world, rank=rank, process_group=dist.group.WORLD) if tp > 1 else dict(tp=1, rank=0)
    m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=4096, seed=9, fused=5, shard_from_full=True, **kw)
    m.capture()
    m.reset_state()
    toks = [int(m.prefill(prompt, chunk=128))]
    ok = int(m.pos) == prompt.shape[1]
    for _ in range(23):
        m.decode()
        toks.append(int(m.next_tok))
    torch.cuda.synchronize()
    res[tp] = (toks, ok)
    if rank == 0:
        print(f"tp={tp}", toks, "pos ok" if ok else "pos WRONG", flush=True)
if rank == 0:
    a, b = res[1][0], res[world][0]
    agree = sum(int(x == y) for x, y in zip(a, b))
    if a[:4] == b[:4] and agree >= 22 and res[1][1] and res[world][1]:
        print("PREFILL-TP AGREE", agree, "of", len(a), flush=True)
    else:
        print("PREFILL-TP DISAGREE", agree, "of", len(a), flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0)
