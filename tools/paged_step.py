"""Paged against contiguous KV cache on one GPU: the tools/ragged_step.py setup (Llama-3.1-8B shape, 32 layers, 4-bit, gs 64, fp16,
batch 32, cache_len 8192, ragged, fused=True, positions uniform in [0, 8192)), the paged and the unpaged model in one process, measured
alternately.  For each --kv-bits it prints JSON lines with
  - "positions": decode step time and layer 0's attention launch (CUDA events, median over --reps alternations), the packed
    prefill of 32 prompts with lengths uniform in [16, 1024], and the cache bytes the slots hold (pages in use x page bytes) against
    the contiguous caches' bytes -- that last figure is arithmetic, not a measurement;
  - "fork": the same for 32 slots forked from one 4096-token prefix (one prefill, 31 forks);
  - the GPU name, power limit and median SM clock over the run (read-only nvidia-smi queries).

    python tools/paged_step.py [--kv-bits 16,8,4] [--kv-group-size 64] [--steps 20] [--reps 3]"""
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
from hqq_b200 import harness  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402
from ragged_step import timed  # noqa: E402

B, L = 32, 8192


def attention_once(m, dev):
    """Layer 0's attention launch of the fused step, as step_fused issues it."""
    lib, s, b = load(), m.shape, m._bufs
    code, st, blk = DTYPE_CODE[m.dtype], stream_ptr(dev), m.blocks[0]
    if m.attn_kernel != "single":
        m._attn_split(lib, blk, s.n_heads, s.n_kv_heads, code, st)
    elif m.kv_pages is not None:
        check(lib.hqq_b200_glue_rope_attn_decode_batch_paged(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(m.cos), ptr(m.sin), ptr(blk["k_cache"]),
                                                             ptr(blk["v_cache"]), ptr(m.page_table), ptr(m.pos), ptr(b["a"]), s.n_heads, s.n_kv_heads, L,
                                                             s.head_dim, B, m.kv_pages, code, st))
    else:
        check(lib.hqq_b200_glue_rope_attn_decode_batch_seqpos(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(m.cos), ptr(m.sin), ptr(blk["k_cache"]),
                                                              ptr(blk["v_cache"]), ptr(m.pos), ptr(b["a"]), s.n_heads, s.n_kv_heads, L, s.head_dim, B, code, st))


def place(m, pos, fork_from=None):
    """Empty caches with slot b at position pos[b]; with kv_pages the rows [0, pos[b]) are backed by pages (fork_from: slot 0's pages
    shared by every other slot, as fork() leaves them)."""
    m.reset_state()
    if m.kv_pages is not None:
        if fork_from is None:
            m._apply_pages(m.pages.prefill({b: (0, p) for b, p in enumerate(pos) if p > 0}))
        else:
            m._apply_pages(m.pages.prefill({0: (0, fork_from)}))
            for d in range(1, B):
                m.fork(0, d)
    m.pos.copy_(torch.as_tensor(pos, device=m.device))


def held_bytes(m):
    if m.kv_pages is None:
        return m.kv_cache_bytes()
    return (m.kv_pages - m.free_pages) * m.kv_cache_bytes() // (m.kv_pages + 1)


def measure(m, dev, pos, steps, fork_from=None):
    place(m, pos, fork_from)
    for _ in range(3):
        m.decode()
    place(m, pos, fork_from)
    step_ms = timed(dev, m.decode, steps)
    held = held_bytes(m)
    place(m, pos, fork_from)
    attention_once(m, dev)
    attn_ms = timed(dev, lambda: attention_once(m, dev), steps)
    return step_ms, attn_ms, held


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv-bits", default="16,8", help="any of 16, 8 and 4")
    ap.add_argument("--kv-group-size", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    shape = harness.LLAMA31_8B
    g = torch.Generator().manual_seed(1)
    pos = torch.randint(0, L - args.steps - 4, (B,), generator=g).tolist()  # as tools/ragged_step.py draws them
    lengths = torch.randint(16, 1025, (B,), generator=g).tolist()
    prompts = [torch.randint(0, shape.vocab, (n,), generator=g).to(dev) for n in lengths]
    prefix = 4096
    # pages for the positions and the timed steps, or for the fork and its steps; whichever is more
    n_pages = max(sum(-(-(p + args.steps + 8) // harness.KV_PAGE) for p in pos), prefix // harness.KV_PAGE + 2 * B) + 8
    sampler = ClockSampler(0)
    sampler.start()
    for kb in [int(x) for x in args.kv_bits.split(",")]:
        models = {}
        for name, kw in (("contiguous", {}), ("paged", {"kv_pages": n_pages})):
            m = harness.DecodeModel(shape, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L, fused=True, batch=B, kv_bits=kb,
                                    kv_group_size=args.kv_group_size, ragged=True, **kw)
            m.capture(warmup=2)
            models[name] = m
        res = {name: {"positions": [], "fork": [], "prefill": []} for name in models}
        for _ in range(args.reps):
            for name, m in models.items():  # alternate
                res[name]["positions"].append(measure(m, dev, pos, args.steps))
                res[name]["fork"].append(measure(m, dev, [prefix] * B, args.steps, fork_from=prefix))
                m.reset_state()
                m.prefill(prompts[:2] + [None] * (B - 2), chunk=1024)  # warm-up
                m.reset_state()
                res[name]["prefill"].append(timed(dev, lambda: m.prefill(prompts, chunk=1024)))
        for case in ("positions", "fork"):
            out = {"case": case, "kv_bits": kb, "batch": B, "cache_len": L, "attn_kernel": models["paged"].attn_kernel, "kv_pages": n_pages}
            if case == "positions":
                out.update(pos_mean=round(statistics.mean(pos), 1), pos_max=max(pos))
            else:
                out.update(prefix=prefix)
            for name in models:
                r = res[name][case]
                out[f"{name}_step_ms"] = round(statistics.median(x[0] for x in r), 4)
                out[f"{name}_attn_ms"] = round(statistics.median(x[1] for x in r), 4)
                out[f"{name}_cache_bytes_held"] = r[-1][2]
                if case == "positions":
                    out[f"{name}_prefill_packed_ms"] = round(statistics.median(res[name]["prefill"]), 3)
            out["held_fraction"] = round(out["paged_cache_bytes_held"] / out["contiguous_cache_bytes_held"], 4)
            print(json.dumps({**out, **info}), flush=True)
        del models, m
        torch.cuda.empty_cache()
    print(json.dumps({"clocks": sampler.stop(), **info}), flush=True)


if __name__ == "__main__":
    main()
