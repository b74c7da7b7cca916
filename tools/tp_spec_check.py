"""2+ GPU check of tensor-parallel speculative decoding: a tp-way model cut from the full quantised weights (shard_from_full), batch 4,
ragged=True, spec_k=3, runs a packed prefill of prompts of 1, 37, 300 and 120 tokens, then 16 decode_spec() calls with prompt-lookup
drafts interleaved with decode() steps, against the one-GPU model of the same weights.  The verify pass sums the row-parallel outputs
with NCCL and picks targets with the MAX / MIN all-reduces; the emitted tokens must agree on the first calls and in all but two
positions.  Run once with the fp16 cache and once with the 8-bit cache.

    torchrun --nproc-per-node 2 tools/tp_spec_check.py"""
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
prompts = [torch.randint(0, 64, (n,), generator=g, device=dev) for n in (1, 37, 300, 120)]  # small alphabet: lookups hit
for kv_bits in (16, 8):
    res = {}
    for tp in (1, world):
        kw = dict(tp=world, rank=rank, process_group=dist.group.WORLD) if tp > 1 else dict(tp=1, rank=0)
        m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=4096, seed=9, fused=True, batch=4, ragged=True, spec_k=3,
                                kv_bits=kv_bits, shard_from_full=True, **kw)
        m.capture()
        m.capture_spec()
        m.reset_state()
        streams = [[t] for t in m.prefill(prompts, chunk=128).tolist()]
        for i in range(24):
            if i % 3 == 2:
                m.decode()
                for b, t in enumerate(m.tok.tolist()):
                    streams[b].append(t)
            else:
                toks, n_new = m.decode_spec()
                for b in range(4):
                    streams[b] += toks[b, :int(n_new[b])].tolist()
        torch.cuda.synchronize()
        res[tp] = streams
        if rank == 0:
            print(f"kv_bits={kv_bits} tp={tp} lengths", [len(s) for s in streams], "pos", m.pos.tolist(), flush=True)
        del m
        torch.cuda.empty_cache()
    if rank == 0:
        a, b = res[1], res[world]
        n = [min(len(x), len(y)) for x, y in zip(a, b)]
        agree = [sum(int(p == q) for p, q in zip(x, y)) for x, y in zip(a, b)]
        ok = all(x[:4] == y[:4] for x, y in zip(a, b)) and all(ag >= k - 2 for ag, k in zip(agree, n))
        print("SPEC-TP", f"kv_bits={kv_bits}", "AGREE" if ok else "DISAGREE", agree, "of", n, flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0)
