"""2+ GPU check of sampling under tensor parallelism: a tp-way model with do_sample (fused=5 with the peer-memory exchange, and a
lock-step batch of 2 on the 8-launch path with NCCL) runs prefill + 16 sampled steps.  Every rank must pick the same token at every
step, and that token must be sample_tokens on the gathered full-vocabulary logits.  Exits 1 on a mismatch.

    python -m torch.distributed.run --nproc_per_node=2 tools/tp_sample_check.py"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hqq_b200 import harness  # noqa: E402

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
dist.init_process_group("nccl", device_id=dev)
shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
ok = True
for fused, batch in ((5, 1), (True, 2)):
    m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=512, seed=9, fused=fused, batch=batch, tp=world, rank=rank,
                            process_group=dist.group.WORLD, do_sample=True, temperature=0.8, top_k=50, top_p=0.9, sample_seed=77)
    m.capture()
    m.reset_state()
    prompt = torch.randint(0, shape.vocab, (batch, 40), generator=torch.Generator(device=dev).manual_seed(5), device=dev)
    m.prefill(prompt, chunk=16)
    for step in range(16):
        ctr = m._sample_ctr.clone()
        m.decode()
        torch.cuda.synchronize()
        g = torch.empty(world * batch, m.vocab_shard, dtype=m.dtype, device=dev)
        dist.all_gather_into_tensor(g, m._bufs["logits"])
        full = g.view(world, batch, m.vocab_shard).transpose(0, 1).reshape(batch, shape.vocab)
        want = harness.sample_tokens(full, 0.8, 50, 0.9, 77, ctr)
        toks = torch.empty(world * batch, dtype=torch.long, device=dev)
        dist.all_gather_into_tensor(toks, m.next_tok)
        same = bool((toks.view(world, batch) == m.next_tok.view(1, batch)).all())
        exact = torch.equal(want, m.next_tok)
        ok &= same and exact
        if rank == 0 and not (same and exact):
            print(f"fused={fused} batch={batch} step {step}: ranks {toks.tolist()} restatement {want.tolist()}", flush=True)
    if rank == 0:
        print(f"fused={fused} batch={batch}: {'SAME TOKENS ON EVERY RANK' if ok else 'MISMATCH'}", flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0 if ok else 1)
