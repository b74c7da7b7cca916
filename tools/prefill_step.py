"""Prompt prefill on one GPU: the Llama-3.1-8B-shaped model (4-bit, gs 64, fp16) with a 131072-position KV cache, fused=5.  For each
prompt length it prints one JSON line with
  - the prefill (DecodeModel.prefill, chunked): total time and prompt tokens/s (CUDA events around the call),
  - the attention launches of that prefill alone (the same chunks and layers replayed over the filled caches, CUDA events) and
    the rest (total - attention), attention TFLOP/s with FLOPs = 4 * 128 * n_q * sum(positions attended) per layer, against 989,
  - F.scaled_dot_product_attention on the same shapes in the same run: one causal call per layer over the whole prompt (q [1, 32,
    T, 128], k / v expanded to 32 heads; the same positions attended, so the same FLOPs),
  - the GPU name, power limit and median SM clock over the run (read-only nvidia-smi queries).
A last line times 8192 one-token decode steps from position 0 (the captured step), the other way to take in an 8192-token prompt.
With --kv-bits 16,8,4 one model per cache kind is built in the same process and the kinds alternate at every prompt length; for the
8- and 4-bit caches (groups of --kv-group-size) the attention launches read the staging pair, and the staging dequantisation (rows
[0, pos0) of every layer and chunk: hqq_b200_dequantize for 8 bits, hqq_b200_glue_kv4_stage for 4) is timed the same way and reported
as its share of the prefill.  kv_cache_bytes() of each model is printed, and at the end the relative L2 of each quantised kind's
last-position logits against the 16-bit cache's after one --logits-prompt-token prompt, in fp16 and in bf16.

    python tools/prefill_step.py [--lengths 512,2048,...] [--chunk 4096] [--sdpa-max 131072] [--kv-bits 16,8,4] [--kv-group-size 64]"""
import argparse
import ctypes
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
    ap.add_argument("--kv-bits", default="16")
    ap.add_argument("--kv-group-size", type=int, default=64)
    ap.add_argument("--logits-prompt", type=int, default=4096, help="with two cache kinds: their last-position logits after a prompt this long")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    shape = harness.LLAMA31_8B
    models = {}
    for kb in [int(x) for x in args.kv_bits.split(",")]:
        models[kb] = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=args.cache_len, fused=5, kv_bits=kb,
                                         kv_group_size=args.kv_group_size)
        models[kb].capture(warmup=2)
        print(json.dumps({"kv_bits": kb, "kv_cache_bytes": models[kb].kv_cache_bytes(), **info}), flush=True)
    model = models[min(models)]
    lib, code = load(), DTYPE_CODE[model.dtype]
    hd, hq, hkv, nl = shape.head_dim, shape.n_heads, shape.n_kv_heads, len(model.blocks)
    g = torch.Generator(device=dev).manual_seed(1)
    sampler = ClockSampler(0)
    sampler.start()
    for m in models.values():
        m.reset_state()
        m.prefill(torch.randint(0, shape.vocab, (1, 512), generator=g, device=dev), chunk=args.chunk)  # warm-up: modules, routes
    for T in [int(x) for x in args.lengths.split(",")]:
        prompt = torch.randint(0, shape.vocab, (1, T), generator=g, device=dev)
        for kb, m in models.items():
            m.reset_state()
            total_ms = timed(dev, lambda: m.prefill(prompt, chunk=args.chunk))
            # the same attention launches over the caches the prefill filled (kv8: the staging pair)
            qr = torch.randn(min(T, args.chunk), hq * hd, generator=g, device=dev).half()
            out = torch.empty_like(qr)
            chunks = [(c0, min(args.chunk, T - c0)) for c0 in range(0, T, args.chunk)]
            kc, vc = m._kv8_stage if kb != 16 else (None, None)

            def attention():
                for c0, n in chunks:
                    for blk in m.blocks:
                        check(lib.hqq_b200_glue_attn_prefill(ptr(qr), ptr(blk["k_cache"] if kc is None else kc), ptr(blk["v_cache"] if vc is None else vc),
                                                             ptr(out), c0, n, hq, hkv, args.cache_len, hd, 1, code, stream_ptr(dev)))
            attention()
            attn_ms = timed(dev, attention)
            flops = 4.0 * hd * hq * (T * (T + 1) // 2) * nl
            line = {"prompt_len": T, "kv_bits": kb, "chunk": args.chunk, "cache_len": args.cache_len, "prefill_ms": round(total_ms, 2),
                    "prompt_tok_s": round(T / total_ms * 1e3, 1), "attn_ms": round(attn_ms, 2), "rest_ms": round(total_ms - attn_ms, 2),
                    "attn_share": round(attn_ms / total_ms, 3), "attn_tflops": round(flops / attn_ms / 1e9, 1),
                    "attn_frac_of_989": round(flops / attn_ms / 1e9 / PEAK_TFLOPS, 3)}
            if kb != 16:  # the staging dequantisation of rows [0, c0) the prefill ran before each chunk's attention
                def staging():
                    for c0, n in chunks:
                        if c0 == 0:
                            continue
                        for blk in m.blocks:
                            if kb == 4:
                                check(lib.hqq_b200_glue_kv4_stage(*[ptr(blk[c]) for c in ("k_cache", "k_scale", "k_zero", "v_cache", "v_scale", "v_zero")],
                                                                  ptr(kc), ptr(vc), (ctypes.c_int * 1)(c0), (ctypes.c_int * 1)(n), hkv, args.cache_len, hd,
                                                                  m.kv_group_size, 1, code, stream_ptr(dev)))
                                continue
                            for h in range(hkv):
                                for c, dst in (("k", kc), ("v", vc)):
                                    check(lib.hqq_b200_dequantize(ptr(blk[c + "_cache"][0, h]), ptr(blk[c + "_scale"][0, h]), ptr(blk[c + "_zero"][0, h]),
                                                                  ptr(dst[0, h]), c0, hd, m.kv_group_size, 8, 1, code, stream_ptr(dev)))
                st_ms = timed(dev, staging)
                line.update({"staging_ms": round(st_ms, 2), "staging_share": round(st_ms / total_ms, 4)})
            if kb == 16 and T <= args.sdpa_max:
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
    if args.logits_prompt and len(models) > 1:
        # last-position logits of each quantised cache against the fp16 / bf16 cache after the same prompt, same weights (seed)
        del models, model
        torch.cuda.empty_cache()
        prompt = torch.randint(0, shape.vocab, (1, args.logits_prompt), generator=g, device=dev)
        for dt in (torch.float16, torch.bfloat16):
            logits = {}
            kinds = sorted({16} | {int(x) for x in args.kv_bits.split(",")}, reverse=True)
            for kb in kinds:
                m = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=dt, device=dev, cache_len=args.logits_prompt, fused=5, kv_bits=kb,
                                        kv_group_size=args.kv_group_size)
                m.prefill(prompt, chunk=args.chunk)
                logits[kb] = m.last_logits.float().clone()
                del m
                torch.cuda.empty_cache()
            for kb in kinds[1:]:
                rel = float((logits[kb] - logits[16]).norm() / logits[16].norm())
                print(json.dumps({"logits_prompt": args.logits_prompt, "dtype": str(dt).split(".")[-1], f"kv{kb}_vs_kv16_logits_rel_l2": rel,
                                  "same_argmax": bool(torch.equal(logits[kb].argmax(-1), logits[16].argmax(-1))), **info}), flush=True)


if __name__ == "__main__":
    main()
