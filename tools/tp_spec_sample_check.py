"""2+ GPU check of tensor-parallel sampled speculative decoding (do_sample, sample_keys="position", spec_k=3): a tp-way model, batch 4,
ragged, runs a packed prefill of prompts of 1, 37, 300 and 120 tokens, then 16 decode_spec() calls with prompt-lookup drafts
interleaved with decode() steps.  Every rank must emit the same tokens, and every verify's targets must equal sample_tokens (the
tp = 1 restatement) on the verify's logits gathered from all ranks, at each row's slot, position and sequence number.  Run once with
the fp16 cache and once with the 8-bit cache.

    torchrun --nproc-per-node 2 tools/tp_spec_sample_check.py"""
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
ok = True
for kv_bits in (16, 8):
    m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=4096, seed=9, fused=True, batch=4, ragged=True, spec_k=3,
                            kv_bits=kv_bits, tp=world, rank=rank, process_group=dist.group.WORLD, do_sample=True, sample_keys="position",
                            temperature=0.6, top_k=5, sample_seed=3)
    m.capture()
    m.capture_spec()
    m.reset_state()
    streams = [[t] for t in m.prefill(prompts, chunk=128).tolist()]
    targets_ok = True
    for i in range(24):
        if i % 3 == 2:
            m.decode()
            for b, t in enumerate(m.tok.tolist()):
                streams[b].append(t)
            continue
        pos0 = m.pos.clone()
        toks, n_new = m.decode_spec()
        for b in range(4):
            streams[b] += toks[b, :int(n_new[b])].tolist()
        lg = m.spec_logits.contiguous()  # [4, K + 1, vocab / tp]
        full = torch.empty(world, *lg.shape, dtype=lg.dtype, device=dev)
        dist.all_gather_into_tensor(full, lg)
        full = full.permute(1, 2, 0, 3).reshape(4, 4, -1)  # [batch, K + 1, vocab], shards in rank order
        tg = m._spec_targets.view(4, 4)
        for t in range(4):
            ref = harness.sample_tokens(full[:, t], m.temperature, m.top_k, m.top_p, m.sample_seed, harness.position_counter(pos0 + t, m.seq))
            targets_ok &= torch.equal(ref, tg[:, t])
    torch.cuda.synchronize()
    lens = torch.tensor([len(s) for s in streams], device=dev)
    flat = torch.tensor(sum(streams, []), device=dev)
    every = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(every, flat)
    same = all(torch.equal(e, flat) for e in every)
    if rank == 0:
        print("SPEC-SAMPLE-TP", f"kv_bits={kv_bits} tp={world}", "ranks", "AGREE" if same else "DISAGREE", "targets",
              "MATCH" if targets_ok else "MISMATCH", "lengths", lens.tolist(), flush=True)
    ok &= same and targets_ok
    del m
    torch.cuda.empty_cache()
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0 if ok else 1)
