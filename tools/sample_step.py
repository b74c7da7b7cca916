"""Cost of sampling in the captured decode step: the Llama-3-8B-shaped model (4-bit, gs 64, fp16, fused=5, batch 1) at position
--pos, one model per variant, the variants alternating round by round in one process:
  greedy, T 0.6 / top_k 5, T 1 / top_p 0.9, T 0.7 / top_k 50 / top_p 0.95.
Prints JSON lines with
  - each variant's step time (median over --rounds rounds of --steps graph replays, CUDA events),
  - the head's last launch alone on the model's own logits: hqq_b200_glue_argmax against hqq_b200_glue_sample per variant (and
    T 1 without a filter), each captured --launches times in one graph and replayed once, per-launch microseconds,
  - batch 32: the sampling launch over 32 rows against torch.argmax over them (the greedy batched head), and the step of a batch-32
    model (fused=True) greedy against T 0.7 / top_k 50 / top_p 0.95,
  - the GPU name, power limit and median SM clock of the run (read-only nvidia-smi queries).

    python tools/sample_step.py [--pos 1024] [--steps 100] [--rounds 5] [--launches 1000]"""
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
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402

VARIANTS = {"greedy": None, "T0.6/k5": (0.6, 5, 1.0), "T1/p0.9": (1.0, 0, 0.9), "T0.7/k50/p0.95": (0.7, 50, 0.95)}


def graph_us(dev, fn, launches):
    """fn() enqueues one launch; `launches` of them in one graph, replayed once after a warm replay: microseconds per launch."""
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            fn()
    g.replay()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) * 1e3 / launches


def step_ms(model, pos, steps):
    dev = model.device
    model.tok.fill_(7)
    model.pos.fill_(pos)
    for _ in range(3):
        model.decode()
    model.pos.fill_(pos)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        model.decode()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / steps


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
    shape, lib, code = harness.LLAMA3_8B, load(), DTYPE_CODE[torch.float16]
    models = {}
    for name, v in VARIANTS.items():
        kw = {} if v is None else dict(do_sample=True, temperature=v[0], top_k=v[1], top_p=v[2], sample_seed=1)
        m = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=args.cache_len, fused=5, **kw)
        m.capture(warmup=2)
        models[name] = m
    sampler = ClockSampler(0)
    sampler.start()
    times = {n: [] for n in models}
    for _ in range(args.rounds):
        for name, m in models.items():
            times[name].append(step_ms(m, args.pos, args.steps))
    g_ms = statistics.median(times["greedy"])
    for name in models:
        ms = statistics.median(times[name])
        print(json.dumps({"variant": name, "batch": 1, "pos": args.pos, "step_ms": round(ms, 4), "tok_s": round(1e3 / ms, 1),
                          "over_greedy_us": round((ms - g_ms) * 1e3, 1), "rounds_ms": [round(t, 4) for t in times[name]]}), flush=True)
    # the head's last launch alone, on the greedy model's own logits after a step at pos
    st = lambda: stream_ptr(dev)  # noqa: E731  (read at call time: under capture it is the capturing stream)
    logits = models["greedy"]._bufs["logits"]
    out = torch.zeros(32, dtype=torch.long, device=dev)
    ctr = torch.zeros(1, dtype=torch.long, device=dev)
    launch = {"argmax": lambda: check(lib.hqq_b200_glue_argmax(ptr(logits), shape.vocab, ptr(out), code, st()))}
    for name, v in list(VARIANTS.items())[1:] + [("T1", (1.0, 0, 1.0))]:
        launch[name] = (lambda v=v, x=logits, rows=1: check(lib.hqq_b200_glue_sample(ptr(x), shape.vocab, x.stride(0), rows, v[0], v[1], v[2], 1, ptr(ctr),
                                                                                   ptr(out), code, st())))
    for name, fn in launch.items():
        print(json.dumps({"launch": name, "rows": 1, "us_per_launch": round(graph_us(dev, fn, args.launches), 2), "launches": args.launches}), flush=True)
    # batch 32: rows of the same spread as the model's logits
    rows32 = (torch.randn(32, shape.vocab, device=dev, generator=torch.Generator(device=dev).manual_seed(3)) * float(logits.float().std())).half()
    tok32 = torch.zeros(32, dtype=torch.long, device=dev)
    b32 = {"torch.argmax": lambda: torch.argmax(rows32, dim=-1, out=tok32)}
    for name, v in list(VARIANTS.items())[1:]:
        b32[name] = (lambda v=v: check(lib.hqq_b200_glue_sample(ptr(rows32), shape.vocab, shape.vocab, 32, v[0], v[1], v[2], 1, ptr(ctr), ptr(out), code,
                                                                 st())))
    for name, fn in b32.items():
        print(json.dumps({"launch": name, "rows": 32, "us_per_launch": round(graph_us(dev, fn, args.launches // 10), 2),
                          "launches": args.launches // 10}), flush=True)
    del models
    torch.cuda.empty_cache()
    bm = {}
    for name in ("greedy", "T0.7/k50/p0.95"):
        v = VARIANTS[name]
        kw = {} if v is None else dict(do_sample=True, temperature=v[0], top_k=v[1], top_p=v[2], sample_seed=1)
        m = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=args.cache_len, fused=True, batch=32, **kw)
        m.capture(warmup=2)
        bm[name] = m
    bt = {n: [] for n in bm}
    for _ in range(args.rounds):
        for name, m in bm.items():
            bt[name].append(step_ms(m, args.pos, args.steps // 2))
    for name in bm:
        ms = statistics.median(bt[name])
        print(json.dumps({"variant": name, "batch": 32, "pos": args.pos, "step_ms": round(ms, 4), "tok_s": round(32e3 / ms, 1),
                          "over_greedy_us": round((ms - statistics.median(bt["greedy"])) * 1e3, 1)}), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks, **info}), flush=True)


if __name__ == "__main__":
    main()
