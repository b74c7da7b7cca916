"""Speculative verify step against the plain decode steps on one GPU, Llama-3-8B shape (32 layers, 4-bit, gs 64, fp16), fp16 KV cache,
cache_len 33024, at positions 1024 and 32768.  Prints JSON lines, each with the GPU name and power limit read in the same process:
  - "verify": the captured verify step (decode_spec's graph, drafts -1) for K in --ks at batch 1 and 8, and per accepted count
    a + 1 in 1 .. K + 1 the time per emitted token, step_ms / (a + 1);
  - "ragged_step": the captured ragged decode step (spec_k unset) at batch 1 and 8;
  - "fused5_step": the batch-1 one-token step (fused=5) bench.py times;
  - "ngram": hqq_b200_glue_ngram_draft at position 131071, batch 32.
The break-even acceptance against a plain step is the smallest a + 1 whose time per token is below it.  All times are CUDA events over
--steps replays after warm-up, medians of --reps windows.

    python tools/spec_step.py [--ks 1,2,3,4,7] [--steps 20] [--reps 3]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import check, load, ptr, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402
from ragged_step import timed  # noqa: E402

L = 33024  # > 32768 + 8, a multiple of 64
POSITIONS = (1024, 32768)


def median_ms(dev, fn, steps, reps, reset):
    out = []
    for _ in range(reps):
        reset()
        fn()
        reset()
        out.append(timed(dev, fn, steps))
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,3,4,7")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    shape = harness.LLAMA3_8B
    base = dict(nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L)
    with torch.no_grad():
        m = harness.DecodeModel(shape, **base)  # fused=5, batch 1, as bench.py
        m.capture(warmup=2)
        for p in POSITIONS:
            ms = median_ms(dev, m.graph.replay, args.steps, args.reps, lambda: m.pos.fill_(p))
            print(json.dumps({"case": "fused5_step", "pos": p, "batch": 1, "step_ms": round(ms, 4), **info}), flush=True)
        del m
        torch.cuda.empty_cache()
        for B in [int(x) for x in args.batches.split(",")]:
            plain = {}
            for k in [None] + [int(x) for x in args.ks.split(",")]:
                m = harness.DecodeModel(shape, **base, batch=B, ragged=True, fused=True, spec_k=k)
                m.capture(warmup=2)
                if k is None:
                    for p in POSITIONS:
                        plain[p] = median_ms(dev, m.graph.replay, args.steps, args.reps, lambda: m.pos.fill_(p))
                        print(json.dumps({"case": "ragged_step", "pos": p, "batch": B, "step_ms": round(plain[p], 4), **info}), flush=True)
                else:
                    m.capture_spec(warmup=2)
                    for p in POSITIONS:
                        ms = median_ms(dev, m.spec_graph.replay, args.steps, args.reps, lambda: (m.pos.fill_(p), m._spec_drafts.fill_(-1)))
                        per = {a1: round(ms / a1, 4) for a1 in range(1, k + 2)}
                        even = next((a1 for a1 in range(1, k + 2) if ms / a1 < plain[p]), None)
                        print(json.dumps({"case": "verify", "K": k, "pos": p, "batch": B, "step_ms": round(ms, 4), "ms_per_token_by_emitted": per,
                                          "ragged_step_ms": round(plain[p], 4), "break_even_emitted": even, **info}), flush=True)
                del m
                torch.cuda.empty_cache()
        # the n-gram kernel alone: 32 slots at position 131071 over random histories of a small alphabet
        B, Lh, K = 32, 131072, 7
        g = torch.Generator(device=dev).manual_seed(1)
        hist = torch.randint(0, 64, (B, Lh), generator=g, device=dev, dtype=torch.int32)
        pos = torch.full((B,), Lh - 1, dtype=torch.long, device=dev)
        tok = torch.randint(0, 64, (B,), generator=g, device=dev)
        drafts = torch.empty(B, K, dtype=torch.long, device=dev)
        lib, st = load(), stream_ptr(dev)
        run = lambda: check(lib.hqq_b200_glue_ngram_draft(ptr(hist), ptr(pos), ptr(tok), ptr(drafts), Lh, K, B, st))
        ms = median_ms(dev, run, 50, args.reps, lambda: None)
        print(json.dumps({"case": "ngram", "pos": Lh - 1, "batch": B, "K": K, "kernel_us": round(ms * 1000, 2), **info}), flush=True)


if __name__ == "__main__":
    main()
