"""Prompt prefill on one GPU: the Llama-3.1-8B-shaped model (4-bit, gs 64, fp16) with a 131072-position KV cache, fused=5.  For each
prompt length it prints one JSON line with
  - the prefill (DecodeModel.prefill, chunked): total time and prompt tokens/s (CUDA events around the call),
  - the attention launches of that prefill alone (the same chunks and layers replayed over the filled caches, CUDA events) and
    the rest (total - attention), attention TFLOP/s with FLOPs = 4 * 128 * n_q * sum(positions attended) per layer, against 989,
  - F.scaled_dot_product_attention on the same shapes in the same run: one causal call per layer over the whole prompt (q [1, 32,
    T, 128], k / v expanded to 32 heads; the same positions attended, so the same FLOPs),
  - the GPU name, power limit and median SM clock over the run (read-only nvidia-smi queries).
A last line times 8192 one-token decode steps from position 0 (the captured step), the other way to take in an 8192-token prompt.

    python tools/prefill_step.py [--lengths 512,2048,...] [--chunk 4096] [--sdpa-max 131072]"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler  # noqa: E402
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense fp16


def timed(dev, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", default="512,2048,8192,32768,131072")
    ap.add_argument("--chunk", type=int, default=4096)
    ap.add_argument("--cache-len", type=int, default=131072)
    ap.add_argument("--sdpa-max", type=int, default=131072, help="longest prompt the SDPA comparison runs on")
    ap.add_argument("--decode-steps", type=int, default=8192)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    shape = harness.LLAMA31_8B
    model = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=args.cache_len, fused=5)
    model.capture(warmup=2)
    lib, code = load(), DTYPE_CODE[model.dtype]
    hd, hq, hkv, nl = shape.head_dim, shape.n_heads, shape.n_kv_heads, len(model.blocks)
    g = torch.Generator(device=dev).manual_seed(1)
    sampler = ClockSampler(0)
    sampler.start()
    model.reset_state()
    model.prefill(torch.randint(0, shape.vocab, (1, 512), generator=g, device=dev), chunk=args.chunk)  # warm-up: modules, routes
    for T in [int(x) for x in args.lengths.split(",")]:
        prompt = torch.randint(0, shape.vocab, (1, T), generator=g, device=dev)
        model.reset_state()
        total_ms = timed(dev, lambda: model.prefill(prompt, chunk=args.chunk))
        # the same attention launches over the caches the prefill filled
        qr = torch.randn(min(T, args.chunk), hq * hd, generator=g, device=dev).half()
        out = torch.empty_like(qr)
        chunks = [(c0, min(args.chunk, T - c0)) for c0 in range(0, T, args.chunk)]

        def attention():
            for c0, n in chunks:
                for blk in model.blocks:
                    check(lib.hqq_b200_glue_attn_prefill(ptr(qr), ptr(blk["k_cache"]), ptr(blk["v_cache"]), ptr(out), c0, n, hq, hkv, args.cache_len, hd,
                                                         1, code, stream_ptr(dev)))
        attention()
        attn_ms = timed(dev, attention)
        flops = 4.0 * hd * hq * (T * (T + 1) // 2) * nl
        line = {"prompt_len": T, "chunk": args.chunk, "cache_len": args.cache_len, "prefill_ms": round(total_ms, 2),
                "prompt_tok_s": round(T / total_ms * 1e3, 1), "attn_ms": round(attn_ms, 2), "rest_ms": round(total_ms - attn_ms, 2),
                "attn_share": round(attn_ms / total_ms, 3), "attn_tflops": round(flops / attn_ms / 1e9, 1),
                "attn_frac_of_989": round(flops / attn_ms / 1e9 / PEAK_TFLOPS, 3)}
        if T <= args.sdpa_max:
            q = torch.randn(1, hq, T, hd, generator=g, device=dev).half()
            k = torch.randn(1, hkv, T, hd, generator=g, device=dev).half().repeat_interleave(hq // hkv, dim=1)
            v = torch.randn(1, hkv, T, hd, generator=g, device=dev).half().repeat_interleave(hq // hkv, dim=1)
            F.scaled_dot_product_attention(q, k, v, is_causal=True)
            sd_ms = timed(dev, lambda: F.scaled_dot_product_attention(q, k, v, is_causal=True)) * nl
            line.update({"sdpa_ms": round(sd_ms, 2), "sdpa_tflops": round(flops / sd_ms / 1e9, 1), "attn_vs_sdpa": round(sd_ms / attn_ms, 3)})
            del q, k, v
        line.update(info)
        print(json.dumps(line), flush=True)
        del qr, out
    # the captured one-token step, fed from position 0
    model.reset_state()
    model.decode()
    model.reset_state()
    steps = args.decode_steps

    def decode():
        for _ in range(steps):
            model.decode()
    dec_ms = timed(dev, decode)
    print(json.dumps({"decode_steps": steps, "decode_total_ms": round(dec_ms, 1), "decode_tok_s": round(steps / dec_ms * 1e3, 1), **info}), flush=True)
    clocks = sampler.stop()
    print(json.dumps({"clocks": clocks, **info}), flush=True)


if __name__ == "__main__":
    main()
