"""2+ GPU check of per-slot sampling under tensor parallelism: a tp-way model with slot_sampling (fused=5 with the peer-memory
exchange at batch 1, and a lock-step batch of 2 on the 8-launch path with NCCL) runs prefill + 16 steps with a penalised sampled
slot and, at batch 2, a penalised greedy one.  Every rank must pick the same token and hold the same counts at every step, and the
token must be apply_penalties + sample_tokens on the gathered full-vocabulary logits with the counts after the step.  Exits 1 on a
mismatch.

    python -m torch.distributed.run --nproc_per_node=2 tools/tp_slot_sampling_check.py"""
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
                            process_group=dist.group.WORLD, do_sample=True, temperature=0.8, top_k=50, top_p=0.9, sample_seed=77, slot_sampling=True)
    m.capture()
    m.reset_state()
    m.set_sampling(0, repetition_penalty=1.3, frequency_penalty=0.4, presence_penalty=0.2)
    if batch > 1:
        m.set_sampling(1, temperature=0, repetition_penalty=1.5, frequency_penalty=0.1)
    prompt = torch.randint(0, 64, (batch, 40), generator=torch.Generator(device=dev).manual_seed(5), device=dev)
    m.prefill(prompt, chunk=16)
    for step in range(16):
        ctr, before, tok = m._sample_ctr.clone(), m.counts.clone(), m.tok.clone()
        m.decode()
        torch.cuda.synchronize()
        g = torch.empty(world * batch, m.vocab_shard, dtype=m.dtype, device=dev)
        dist.all_gather_into_tensor(g, m._bufs["logits"])
        full = g.view(world, batch, m.vocab_shard).transpose(0, 1).reshape(batch, shape.vocab)
        before[torch.arange(batch, device=dev), tok] += 1
        pen = harness.apply_penalties(full, m.counts, m.prompt_seen, m.slot_repetition, m.slot_frequency, m.slot_presence)
        want = harness.sample_tokens(pen, m.slot_temperature, m.slot_top_k, m.slot_top_p, 77, ctr)
        toks = torch.empty(world * batch, dtype=torch.long, device=dev)
        dist.all_gather_into_tensor(toks, m.next_tok)
        counts = torch.empty(world, batch, shape.vocab, dtype=torch.int32, device=dev)
        dist.all_gather_into_tensor(counts, m.counts)
        same = bool((toks.view(world, batch) == m.next_tok.view(1, batch)).all()) and bool((counts == m.counts.unsqueeze(0)).all())
        exact = torch.equal(want, m.next_tok) and torch.equal(before, m.counts)
        ok &= same and exact
        if rank == 0 and not (same and exact):
            print(f"fused={fused} batch={batch} step {step}: ranks {toks.tolist()} restatement {want.tolist()} counts ok {torch.equal(before, m.counts)}",
                  flush=True)
    if rank == 0:
        print(f"fused={fused} batch={batch}: {'SAME TOKENS ON EVERY RANK' if ok else 'MISMATCH'}", flush=True)
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0 if ok else 1)
