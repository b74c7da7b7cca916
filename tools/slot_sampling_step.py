"""Cost of per-slot sampling and penalties in the captured decode step: the Llama-3-8B-shaped model (4-bit, gs 64, fp16) at position
--pos, batch 1 (fused=5) and a ragged batch of 32 (fused=True), one model per variant, the variants alternating round by round:
  greedy; do_sample (T 0.7 / top_k 50 / top_p 0.95); slot_sampling with every slot on those settings and neutral penalties;
  slot_sampling with mixed settings (greedy, T 0.7 / top_p 0.9, T 1 / top_k 50, ... by slot) and repetition 1.1, frequency 0.3,
  presence 0.2.
Prints JSON lines with each variant's step time (median over --rounds rounds of --steps graph replays, CUDA events), the
hqq_b200_glue_penalize launch alone (1 and 32 rows of the full vocabulary, --launches launches captured in one graph, per-launch
microseconds), and the GPU name, power limit and median SM clock of the run (read-only nvidia-smi queries).

    python tools/slot_sampling_step.py [--pos 1024] [--steps 100] [--rounds 5] [--launches 1000]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler  # noqa: E402
from long_context_step import gpu_info  # noqa: E402
from sample_step import graph_us, step_ms  # noqa: E402
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402

SAMPLE = dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.95, sample_seed=1)
VARIANTS = {"greedy": {}, "do_sample": SAMPLE, "slot_neutral": dict(SAMPLE, slot_sampling=True), "slot_mixed": dict(SAMPLE, slot_sampling=True)}
MIXED = [dict(temperature=0), dict(temperature=0.7, top_k=0, top_p=0.9), dict(temperature=1.0, top_k=50, top_p=1.0), dict(temperature=0.6, top_k=5)]


def models(shape, fused, batch, cache_len):
    out = {}
    for name, kw in VARIANTS.items():
        m = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device="cuda", cache_len=cache_len, fused=fused, batch=batch,
                                ragged=batch > 1, **kw)
        m.capture(warmup=2)
        if name == "slot_mixed":
            for b in range(batch):
                m.set_sampling(b, repetition_penalty=1.1, frequency_penalty=0.3, presence_penalty=0.2, **MIXED[b % len(MIXED)])
            m.prompt_seen[:, ::7] = 1  # a prompt's worth of seen tokens
        out[name] = m
    return out


def run(shape, fused, batch, args):
    ms = models(shape, fused, batch, args.cache_len)
    times = {n: [] for n in ms}
    for _ in range(args.rounds):
        for name, m in ms.items():
            times[name].append(step_ms(m, args.pos, args.steps))
    g_ms = statistics.median(times["greedy"])
    for name in ms:
        t = statistics.median(times[name])
        print(json.dumps({"variant": name, "batch": batch, "fused": fused, "pos": args.pos, "step_ms": round(t, 4), "tok_s": round(batch * 1e3 / t, 1),
                          "over_greedy_us": round((t - g_ms) * 1e3, 1), "rounds_ms": [round(x, 4) for x in times[name]]}), flush=True)
    del ms
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pos", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=1000)
    ap.add_argument("--cache-len", type=int, default=2048)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    sampler = ClockSampler(0)
    sampler.start()
    shape = harness.LLAMA3_8B
    run(shape, 5, 1, args)
    run(shape, True, 32, args)
    # the penalize launch alone over rows of the full vocabulary
    lib, code, V = load(), DTYPE_CODE[torch.float16], shape.vocab
    st = lambda: stream_ptr(dev)  # noqa: E731  (read at call time: under capture it is the capturing stream)
    for rows in (1, 32):
        g = torch.Generator(device=dev).manual_seed(rows)
        x = torch.randn(rows, V, device=dev, generator=g).half()
        out = torch.empty_like(x)
        counts = torch.randint(0, 2, (rows, V), device=dev, generator=g, dtype=torch.int32)
        prompt = torch.randint(0, 2, (rows, V), device=dev, generator=g, dtype=torch.uint8)
        tok = torch.zeros(rows, dtype=torch.long, device=dev)
        r, f, p = (torch.full((rows,), v, device=dev) for v in (1.1, 0.3, 0.2))
        fn = lambda: check(lib.hqq_b200_glue_penalize(ptr(x), V, V, rows, 1, ptr(r), ptr(f), ptr(p), ptr(counts), ptr(prompt), ptr(tok), ptr(out), V,  # noqa: E731
                                                      code, st()))
        us = graph_us(dev, fn, args.launches)
        moved = rows * V * (2 + 4 + 1 + 2)  # logits, counts, prompt in; rows out
        print(json.dumps({"launch": "penalize", "rows": rows, "us_per_launch": round(us, 2), "launches": args.launches,
                          "GB_s": round(moved / us / 1e3, 1)}), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks, **info}), flush=True)


if __name__ == "__main__":
    main()
