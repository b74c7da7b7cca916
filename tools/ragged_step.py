"""Ragged batches on one GPU: the Llama-3.1-8B-shaped model (32 layers, 4-bit, gs 64, fp16), batch 32, cache_len 8192, fused=True.
For each --kv-bits it prints JSON lines with
  - decode: the captured step of a ragged model whose 32 sequences sit at positions drawn uniformly from [0, 8192), against
    lock-step models at the largest and at the mean of those positions: whole-step time and the attention launch alone (layer 0,
    replayed; CUDA events);
  - prefill of 32 prompts with lengths uniform in [16, 1024]: one packed variable-length prefill, one slot at a time (32 refill
    calls), and the lock-step prefill of 32 prompts of the longest length (the cost of padding every prompt to it);
  - the GPU name, power limit and median SM clock over the run (read-only nvidia-smi queries).
The ragged and lock-step models are built one after the other (the fp16 caches of one take 34 GB).

    python tools/ragged_step.py [--kv-bits 16,8] [--steps 20]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler  # noqa: E402
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402

B, L = 32, 8192


def timed(dev, fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / reps


def attention_once(m, dev):
    """Layer 0's attention launch of the fused step, as step_fused issues it."""
    lib, s, b = load(), m.shape, m._bufs
    code, st, blk = DTYPE_CODE[m.dtype], stream_ptr(dev), m.blocks[0]
    if m.attn_kernel != "single":
        m._attn_split(lib, blk, s.n_heads, s.n_kv_heads, code, st)
        return
    fn = lib.hqq_b200_glue_rope_attn_decode_batch_seqpos if m.ragged else lib.hqq_b200_glue_rope_attn_decode_batch
    check(fn(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(m.cos), ptr(m.sin), ptr(blk["k_cache"]), ptr(blk["v_cache"]), ptr(m.pos), ptr(b["a"]), s.n_heads,
             s.n_kv_heads, L, s.head_dim, B, code, st))


def decode(m, dev, pos, steps):
    """Whole captured step and attention launch (ms) with the sequences at `pos` (replays advance them; the mean over `steps`)."""
    m.pos.copy_(torch.as_tensor(pos, device=dev).view(-1)[: m.pos.numel()])
    for _ in range(3):
        m.decode()
    m.pos.copy_(torch.as_tensor(pos, device=dev).view(-1)[: m.pos.numel()])
    step_ms = timed(dev, m.decode, steps)
    m.pos.copy_(torch.as_tensor(pos, device=dev).view(-1)[: m.pos.numel()])
    attention_once(m, dev)
    attn_ms = timed(dev, lambda: attention_once(m, dev), steps)
    return step_ms, attn_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv-bits", default="16,8")
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    shape = harness.LLAMA31_8B
    g = torch.Generator().manual_seed(1)
    pos = torch.randint(0, L - args.steps - 4, (B,), generator=g)  # uniform in [0, 8192), leaving room for the timed replays
    lengths = torch.randint(16, 1025, (B,), generator=g).tolist()
    prompts = [torch.randint(0, shape.vocab, (n,), generator=g).to(dev) for n in lengths]
    longest = max(lengths)
    padded = torch.randint(0, shape.vocab, (B, longest), generator=g).to(dev)
    sampler = ClockSampler(0)
    sampler.start()
    for kb in [int(x) for x in args.kv_bits.split(",")]:
        res = {"kv_bits": kb, "batch": B, "cache_len": L, "pos_max": int(pos.max()), "pos_mean": round(float(pos.float().mean()), 1),
               "prompt_tokens": sum(lengths), "prompt_longest": longest}
        for ragged in (True, False):
            m = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L, fused=True, batch=B, kv_bits=kb,
                                    ragged=ragged)
            m.capture(warmup=2)
            m.reset_state()
            if ragged:
                res["attn_kernel"] = m.attn_kernel
                res["ragged_step_ms"], res["ragged_attn_ms"] = decode(m, dev, pos, args.steps)
                m.reset_state()
                m.prefill(prompts[:2] + [None] * (B - 2), chunk=1024)  # warm-up
                m.reset_state()
                res["prefill_packed_ms"] = timed(dev, lambda: m.prefill(prompts, chunk=1024))
                m.reset_state()

                def one_by_one():
                    for b in range(B):
                        m.prefill([prompts[b] if i == b else None for i in range(B)], chunk=1024)
                res["prefill_one_slot_at_a_time_ms"] = timed(dev, one_by_one)
            else:
                for name, p in (("max", int(pos.max())), ("mean", int(round(float(pos.float().mean()))))):
                    res[f"lockstep_{name}_step_ms"], res[f"lockstep_{name}_attn_ms"] = decode(m, dev, [p], args.steps)
                m.reset_state()
                m.prefill(padded[:, :64], chunk=1024)  # warm-up
                m.reset_state()
                res["prefill_lockstep_longest_ms"] = timed(dev, lambda: m.prefill(padded, chunk=1024))
            del m
            torch.cuda.empty_cache()
        res = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}
        print(json.dumps({**res, **info}), flush=True)
    print(json.dumps({"clocks": sampler.stop(), **info}), flush=True)


if __name__ == "__main__":
    main()
