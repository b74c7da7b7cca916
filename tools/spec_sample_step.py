"""Sampled speculative decoding on one GPU, Llama-3.1-8B shape (32 layers, 4-bit, gs 64, fp16), fp16 KV cache, cache_len 4096, with
the reference generator's sampling defaults (temperature 0.6, top_k 5, top_p 1) under position keys.  For batch 1, 4 and 32 and K 3
and 7 it prints one JSON line per configuration, each with the GPU name and power limit read in the same process:
  - verify_ms: the captured verify step (decode_spec's graph) at the prompts' end, drafts -1, and all_accepted_tok_s_per_slot =
    (K + 1) / verify_ms, the rate a slot would reach if every draft were accepted;
  - sample_ms / sample_share: the hqq_b200_glue_sample_pos launch over the verify's B (K + 1) logits rows alone, and its share of
    verify_ms;
  - emitted_per_verify: mean tokens emitted per slot and verify over --calls free-running decode_spec() calls with prompt-lookup
    drafts;
  - tok_s_per_slot for sampled decode_spec(), greedy decode_spec() (its own emitted_per_verify beside it) and plain sampled
    decode(): emitted tokens per slot over the wall time of the calls (a host clock around --calls calls ending in a device sync).
The prompts repeat a short random phrase, so prompt lookup finds drafts.  The weights are random: the acceptance a repetitive prompt
gets here says nothing about real text.  CUDA events and host times are medians of --reps windows.

    python tools/spec_sample_step.py [--batches 1,4,32] [--ks 3,7] [--calls 16] [--reps 3]"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, load, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402
from ragged_step import timed  # noqa: E402

L = 4096
PROMPT = 512
SAMPLE = dict(do_sample=True, sample_keys="position", temperature=0.6, top_k=5, top_p=1.0, sample_seed=1)


def prompts(B, dev):
    g = torch.Generator(device=dev).manual_seed(B)
    out = []
    for _ in range(B):  # a random 24-token phrase repeated, then cut: prompt lookup keeps finding its continuation
        phrase = torch.randint(0, 128256, (24,), generator=g, device=dev)
        out.append(phrase.repeat(PROMPT // 24 + 1)[:PROMPT])
    return out


def run_calls(dev, m, calls, spec):
    """(tokens emitted per slot, wall ms) of `calls` decode_spec() (or decode()) calls from the prompts' end."""
    m.reset_state()
    m.prefill(prompts(m.batch, dev), chunk=512)
    torch.cuda.synchronize(dev)
    n = torch.zeros(m.batch, dtype=torch.long, device=dev)
    t0 = time.perf_counter()
    for _ in range(calls):
        if spec:
            n += m.decode_spec()[1]
        else:
            m.decode()
            n += 1
    torch.cuda.synchronize(dev)
    return n.double().mean().item(), (time.perf_counter() - t0) * 1e3


def median(xs):
    return statistics.median(xs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,32")
    ap.add_argument("--ks", default="3,7")
    ap.add_argument("--calls", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    base = dict(nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L, ragged=True, fused=True)
    lib, st = load(), stream_ptr(dev)
    with torch.no_grad():
        for B in [int(x) for x in args.batches.split(",")]:
            for K in [int(x) for x in args.ks.split(",")]:
                rec = {"case": "spec_sample", "batch": B, "K": K, "prompt": PROMPT, "calls": args.calls,
                       "note": "random weights, repetitive prompts: the acceptance says nothing about real text"}
                for mode in ("sampled", "greedy"):
                    m = harness.DecodeModel(harness.LLAMA3_8B, **base, batch=B, spec_k=K, **(SAMPLE if mode == "sampled" else {}))
                    m.capture(warmup=2)
                    m.capture_spec(warmup=2)
                    runs = [run_calls(dev, m, args.calls, True) for _ in range(args.reps)]
                    em, ms = runs[0][0], median([r[1] for r in runs])
                    rec[f"{mode}_spec_emitted_per_verify"] = round(em / args.calls, 3)
                    rec[f"{mode}_spec_tok_s_per_slot"] = round(em / ms * 1e3, 1)
                    if mode == "sampled":
                        runs = [run_calls(dev, m, args.calls, False) for _ in range(args.reps)]
                        rec["sampled_decode_tok_s_per_slot"] = round(args.calls / median([r[1] for r in runs]) * 1e3, 1)
                        pos0 = m.pos.clone()
                        reset = lambda: (m.pos.copy_(pos0), m._spec_drafts.fill_(-1))
                        verify = []
                        for _ in range(args.reps):
                            reset()
                            m.spec_graph.replay()
                            reset()
                            verify.append(timed(dev, m.spec_graph.replay, 10))
                        rows = m._sample_rows(m._bufs["verify_logits"], m._verify_sample_bufs)
                        out = torch.empty(B * (K + 1), dtype=torch.long, device=dev)
                        once = lambda: m._sample(lib, rows, out, DTYPE_CODE[m.dtype], st, pos=m.pos, T=K + 1)
                        once()
                        samp = median([timed(dev, once, 50) for _ in range(args.reps)])
                        rec["verify_ms"] = round(median(verify), 4)
                        rec["all_accepted_tok_s_per_slot"] = round((K + 1) / median(verify) * 1e3, 1)
                        rec["sample_ms"] = round(samp, 4)
                        rec["sample_share"] = round(samp / median(verify), 4)
                    del m
                    torch.cuda.empty_cache()
                print(json.dumps({**rec, **info}), flush=True)


if __name__ == "__main__":
    main()
