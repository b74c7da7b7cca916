"""Long-context decode on one GPU: the Llama-3.1-8B-shaped model (4-bit, gs 64, fp16) with a 131072-position KV cache (17 GB),
caches filled with random rows so no prompt has to be decoded.  For each position it prints one JSON line with
  - the captured step: time and tok/s over >= 50 graph replays (CUDA events; *pos advances inside the graph),
  - the attention launch alone: the 32 layers' split-KV launches captured in one graph, us per launch and GB/s, where
    bytes = 2 n_kv (pos + 1) 128 * 2 (K and V rows read) + q / k / v / out, against the 3.35 TB/s data sheet,
  - at pos 8191 also the one-CTA-per-head kernel on cache_len 8192 caches, the same way,
  - the GPU name, power limit and median SM clock over the run (read-only nvidia-smi queries).
With --kv-bits 16,8,4 one model per cache kind is built in the same process and the kinds alternate at every position; for the 8- and
4-bit caches (HQQ rows, groups of --kv-group-size) the attention bytes are levels plus scale and zero.  kv_cache_bytes() of each
model is printed first.

    python tools/long_context_step.py [--steps 50] [--positions 1024,8191,...] [--kv-bits 16,8,4] [--kv-group-size 64]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM data sheet


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, plim, mx = [x.strip() for x in r.stdout.strip().split(",")[:3]]
        return {"gpu": name, "power_limit_w": float(plim), "sm_max_mhz": float(mx)}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "error": str(e)[:100]}


def time_graph(dev, fn, reps=20):
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--positions", default="1024,8191,16384,32768,65536,131000")
    ap.add_argument("--cache-len", type=int, default=131072)
    ap.add_argument("--kv-bits", default="16")
    ap.add_argument("--kv-group-size", type=int, default=64)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    shape = harness.LLAMA31_8B
    lib = load()
    hd, hq, hkv = shape.head_dim, shape.n_heads, shape.n_kv_heads
    g = torch.Generator(device=dev).manual_seed(1)
    models = {}
    for kb in [int(x) for x in args.kv_bits.split(",")]:
        model = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=args.cache_len, fused=5, kv_bits=kb,
                                    kv_group_size=args.kv_group_size)
        model.capture(warmup=2)
        for blk in model.blocks:
            for n in ("k", "v"):
                c = blk[n + "_cache"]
                for i in range(0, c.shape[2], 16384):
                    rows = torch.randn(c[:, :, i:i + 16384].shape[:-1] + (hd,), generator=g, device=dev, dtype=torch.float32).mul_(0.5).half()
                    if kb != 16:
                        lv, sc, ze = harness.kv8_quantize_rows(rows, args.kv_group_size, kb)
                        c[:, :, i:i + 16384].copy_(lv)
                        blk[n + "_scale"][:, :, i:i + 16384].copy_(sc)
                        blk[n + "_zero"][:, :, i:i + 16384].copy_(ze)
                    else:
                        c[:, :, i:i + 16384].copy_(rows)
                    del rows
        for t in (model._bufs["q"], model._bufs["k"], model._bufs["v"]):
            t.copy_(torch.randn(t.shape, generator=g, device=dev))
        models[kb] = model
        print(json.dumps({"kv_bits": kb, "kv_group_size": args.kv_group_size if kb != 16 else None, "kv_cache_bytes": model.kv_cache_bytes(), **info}),
              flush=True)
    code = DTYPE_CODE[torch.float16]
    small = None
    sampler = ClockSampler(0)
    sampler.start()
    for pos in [int(p) for p in args.positions.split(",")]:
        pos = min(pos, args.cache_len - args.steps - 2)
        for kb, model in models.items():
            b = model._bufs
            model.tok.fill_(7)
            model.pos.fill_(pos)
            for _ in range(3):
                model.decode()
            model.pos.fill_(pos)
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                model.decode()
            e1.record()
            torch.cuda.synchronize(dev)
            step_ms = e0.elapsed_time(e1) / args.steps
            # the attention launches of all 32 layers in one graph, at this position
            model.pos.fill_(pos)

            def split(model=model):  # the stream is read at call time: under capture it is the capturing stream
                for blk in model.blocks:
                    model._attn_split(lib, blk, hq, hkv, code, stream_ptr(dev))
            ms = time_graph(dev, split) / len(model.blocks)
            row = hd * 2 if kb == 16 else hd * kb // 8 + 4 * (hd // args.kv_group_size)  # bytes of one cached row of one kv head
            nbytes = 2 * hkv * (pos + 1) * row + (2 * hq + 2 * hkv) * hd * 2
            line = {"pos": pos, "kv_bits": kb, "cache_len": args.cache_len, "step_ms": round(step_ms, 4), "tok_s": round(1e3 / step_ms, 2),
                    "steps_timed": args.steps, "attn_kernel": model.attn_kernel, "attn_us_per_launch": round(ms * 1e3, 2),
                    "attn_GBps": round(nbytes / ms / 1e6, 1), "attn_frac_of_3350": round(nbytes / ms / 1e6 / HBM_GBS, 3),
                    "attn_bytes_per_launch": nbytes, "kv_bytes_per_step": 32 * nbytes}
            if pos == 8191 and kb == 16 and model.attn_kernel == "split":  # the one-CTA-per-head kernel on cache_len 8192 caches
                if small is None:
                    small = [(torch.randn(1, hkv, 8192, hd, generator=g, device=dev).half(), torch.randn(1, hkv, 8192, hd, generator=g, device=dev).half())
                             for _ in model.blocks]
                cos8, sin8 = model.cos[:8192].contiguous(), model.sin[:8192].contiguous()

                def single(model=model, b=b, cos8=cos8, sin8=sin8):
                    for kc, vc in small:
                        check(lib.hqq_b200_glue_rope_attn_decode(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(cos8), ptr(sin8), ptr(kc), ptr(vc),
                                                                 ptr(model.pos), ptr(b["a"]), hq, hkv, 8192, hd, code, stream_ptr(dev)))
                ms1 = time_graph(dev, single) / len(small)
                line["single_us_per_launch"] = round(ms1 * 1e3, 2)
                line["single_GBps"] = round(nbytes / ms1 / 1e6, 1)
                line["split_speedup"] = round(ms1 / ms, 2)
            line.update(info)
            print(json.dumps(line), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks, **info}), flush=True)


if __name__ == "__main__":
    main()
