"""Prompt scoring cost on one GPU, Llama-3-8B shape (4-bit, gs 64, fp16, fp16 KV cache), batch 1, prompts of 512, 2048, 8192 and
32768 tokens.  Prints JSON lines, each with the GPU name and power limit read in the same process:
  - "head": at min(T, 4096) rows of final-norm output, the LSE head (hqq_b200_lm_logprob: wgmma GEMM with the LSE epilogue + the tile
    merge) against torch.matmul logits + F.log_softmax in fp32 + gather on the same rows, and the largest difference of the two
    log-probabilities;
  - "score": DecodeModel.score() against prefill() on the same prompt (chunk 2048), and the difference per prompt token.
Times are CUDA events, medians of --reps calls after one warm-up call.

    python tools/score_step.py [--layers 32] [--reps 3] [--lengths 512,2048,8192,32768]"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402
from ragged_step import timed  # noqa: E402


def median_ms(dev, fn, reps):
    fn()
    return statistics.median(timed(dev, fn) for _ in range(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lengths", default="512,2048,8192,32768")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("score_step.py measures on a CUDA device")
    dev = torch.device("cuda", 0)
    info = gpu_info()
    lengths = [int(x) for x in a.lengths.split(",")]
    L = -(-(max(lengths) + 1) // 64) * 64
    m = harness.DecodeModel(harness.LLAMA3_8B, n_layers=a.layers, dtype=torch.float16, device=dev, cache_len=L, fused=True)
    lib, st, code, s = load(), stream_ptr(dev), DTYPE_CODE[m.dtype], m.shape
    g = torch.Generator(device=dev).manual_seed(0)
    for T in lengths:
        rows = min(T, harness.LOGPROB_ROWS)
        x = torch.randn(rows, s.hidden, generator=g, device=dev).to(m.dtype)
        tg = torch.randint(0, s.vocab, (rows,), generator=g, device=dev)
        lse = torch.empty(2, rows, device=dev)
        ws = torch.empty(lib.hqq_b200_lm_logprob_workspace_bytes(rows, s.vocab), dtype=torch.uint8, device=dev)

        def fused_head():
            check(lib.hqq_b200_lm_logprob(ptr(x), ptr(m.lm_head), ptr(tg), ptr(lse[0]), ptr(lse[1]), ptr(ws), rows, s.vocab, s.hidden, 0, code, st))

        def torch_head():
            return F.log_softmax(torch.matmul(x, m.lm_head.t()).float(), dim=-1).gather(1, tg.view(-1, 1)).view(-1)

        t_f, t_t = median_ms(dev, fused_head, a.reps), median_ms(dev, torch_head, a.reps)
        diff = float((lse[1] - lse[0] - torch_head()).abs().max())
        print(json.dumps({"kind": "head", **info, "rows": rows, "vocab": s.vocab, "lse_head_ms": round(t_f, 3), "torch_head_ms": round(t_t, 3),
                          "max_abs_logp_diff": diff}), flush=True)
        del x, lse, ws
        prompt = torch.randint(0, s.vocab, (T,), generator=g, device=dev)
        t_p = median_ms(dev, lambda: m.prefill(prompt, chunk=2048), a.reps)
        t_s = median_ms(dev, lambda: m.score(prompt, chunk=2048), a.reps)
        print(json.dumps({"kind": "score", **info, "layers": a.layers, "tokens": T, "prefill_ms": round(t_p, 2), "score_ms": round(t_s, 2),
                          "extra_us_per_token": round((t_s - t_p) * 1e3 / T, 3)}), flush=True)


if __name__ == "__main__":
    main()
