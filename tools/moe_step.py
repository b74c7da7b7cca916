"""Mixture-of-experts decode on one GPU: MIXTRAL_8X7B (32 layers, 8 experts, top-2) at 4-bit, gs 64, fp16, cache_len 4096, every
sequence at position 1024, fused=True.  Prints JSON lines with
  - the captured step at batch 1 and in ragged batches of 8 and 32 (the three models share one set of weights, each has its own
    caches), and the dense LLAMA3_8B step at batch 1 (its default one-token path) as the yardstick; variants alternate round by
    round, each time the median over rounds of CUDA-event-timed replays;
  - the bytes each step had to read, computed from shapes and from the per-layer count of experts the router of the timed step
    selected (read back after timing by one eager step from the same state): attention weights, experts hit, router, lm_head, KV
    rows; and the achieved GB/s;
  - layer 0's grouped gate/up launch at batch 1 (two experts: four 14336 x 4096 matrices) next to a linear_fwd_multi launch over
    the same four matrices (the same bytes; at M = 1 that is the one-token kernel, which prefetches under its predecessor);
  - model construction time and resident weight bytes; GPU name, power limit and SM clock (read-only nvidia-smi queries).

    python tools/moe_step.py [--rounds 5] [--steps 10]"""
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
from bench import ClockSampler  # noqa: E402
from hqq_b200 import harness, ops  # noqa: E402
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr  # noqa: E402
from long_context_step import gpu_info  # noqa: E402

L, POS = 4096, 1024
BPW = 0.5 + 2 * 2 / 64  # 4-bit levels + fp16 scale and zero per group of 64


def timed(dev, fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / reps


def sibling(base, batch, dev):
    """A model of `batch` ragged slots over base's weights: its own embedding, head and caches (n_layers=0 builds none), base's blocks'
    weights."""
    s = base.shape
    m = harness.DecodeModel(s, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L, fused=True, batch=batch, ragged=batch > 1,
                            n_layers=0)
    m.embed, m.lm_head, m.final_norm = base.embed, base.lm_head, base.final_norm
    for blk in base.blocks:
        own = {n: t for n, t in blk.items() if not n.endswith(("_cache",))}
        for n in ("k_cache", "v_cache"):
            own[n] = torch.zeros(batch, *blk[n].shape[1:], device=dev, dtype=blk[n].dtype)
        m.blocks.append(own)
    m.n_layers = len(m.blocks)
    m.quantized_weights = base.quantized_weights
    return m


def step_bytes(m, experts_hit):
    """Bytes one step must read: attention weights and router per layer, the experts the router selected, lm_head, KV rows."""
    s, B = m.shape, m.batch
    hd = s.head_dim
    attn = (2 * s.hidden * s.n_heads * hd + 2 * s.hidden * s.n_kv_heads * hd) * BPW
    expert = 3 * s.hidden * s.inter * BPW
    router = s.n_experts * s.hidden * 2 if s.n_experts else 0
    dense_mlp = 0 if s.n_experts else 3 * s.hidden * s.inter * BPW
    kv = 2 * s.n_kv_heads * hd * 2 * (POS + 1) * B
    per_layer = [attn + router + dense_mlp + kv + expert * e for e in experts_hit]
    return sum(per_layer) + s.vocab * s.hidden * 2


def experts_of_step(m, dev):
    """Run one eager fused step from the current state and record, per layer, how many experts received pairs."""
    hits = []
    orig = m._mlp_fused

    def rec(lib, blk, x, b, M, code, st):
        out = orig(lib, blk, x, b, M, code, st)
        if m.shape.n_experts:
            hits.append(int((b["cnt"] > 0).sum()))
        return out
    m._mlp_fused = rec
    try:
        m.step_fused()
        torch.cuda.synchronize(dev)
    finally:
        del m._mlp_fused
    return hits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    sampler = ClockSampler(0)
    sampler.start()
    t0 = time.perf_counter()
    moe = harness.DecodeModel(harness.MIXTRAL_8X7B, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L, fused=True, batch=32,
                              ragged=True)
    torch.cuda.synchronize(dev)
    build_s = time.perf_counter() - t0
    resident = sum(t.numel() * t.element_size() for blk in moe.blocks for n, v in blk.items() if n == "stack" for st in v.values() for t in st)
    resident += sum(l.W_q.numel() + 2 * l.meta["scale"].numel() * 2 for blk in moe.blocks for n in ("q", "k", "v", "o") for l in [blk[n]])
    resident += sum(blk["router"].numel() * 2 for blk in moe.blocks) + moe.lm_head.numel() * 2
    print(json.dumps({"model": "MIXTRAL_8X7B", "construct_s": round(build_s, 1), "resident_weight_bytes": int(resident),
                      "quantized_weights": moe.quantized_weights, **info}), flush=True)
    models = {"moe_b1": sibling(moe, 1, dev), "moe_b8": sibling(moe, 8, dev), "moe_b32": moe,
              "dense_b1": harness.DecodeModel(harness.LLAMA3_8B, nbits=4, group_size=64, dtype=torch.float16, device=dev, cache_len=L)}
    g = torch.Generator().manual_seed(1)
    for m in models.values():
        m.capture(warmup=2)
        m.reset_state()
        m.tok.copy_(torch.randint(0, m.shape.vocab, (m.batch,), generator=g).to(dev))

    def replay(m):
        m.graph.replay()
    times = {k: [] for k in models}
    for _ in range(args.rounds):
        for name, m in models.items():
            m.pos.fill_(POS)
            replay(m)
            m.pos.fill_(POS)
            times[name].append(timed(dev, lambda: replay(m), args.steps))  # pos advances one row per replay
    for name, m in models.items():
        m.pos.fill_(POS + args.steps - 1)  # the last timed replay's state (its cache rows are rewritten with the same values)
        hits = experts_of_step(m, dev) if m.shape.n_experts else [0] * m.n_layers
        ms = statistics.median(times[name])
        nbytes = step_bytes(m, hits)
        res = {"variant": name, "batch": m.batch, "cache_len": L, "pos": POS, "step_ms": round(ms, 4),
               "step_ms_rounds": [round(t, 4) for t in times[name]], "bytes": int(nbytes), "gb_per_s": round(nbytes / ms / 1e6, 1),
               "experts_hit_per_layer": hits if m.shape.n_experts else None, "path": "step_fused5" if m.fused == 5 else "step_fused"}
        print(json.dumps({**res, **info}), flush=True)

    # layer 0's grouped gate/up at batch 1 against linear_fwd_multi over the same four matrices
    m1 = models["moe_b1"]
    lib, blk, b = load(), m1.blocks[0], m1._moe_bufs
    x = torch.randn(1, m1.shape.hidden, device=dev).half()
    check(lib.hqq_b200_glue_moe_route(ptr(x), ptr(blk["router"]), 1, m1.shape.hidden, 8, 2, ptr(b["ids"]), ptr(b["w"]), ptr(b["pair_of"]), ptr(b["off"]),
                                      ptr(b["cnt"]), ptr(b["token"]), ptr(m1._moe_ticket), DTYPE_CODE[torch.float16], stream_ptr(dev)))
    sel = b["ids"].view(-1).tolist()
    st = blk["stack"]
    grouped = lambda: ops.linear_fwd_grouped(x, b["token"], (st["gate"], st["up"]), [b["gate"], b["up"]], b["off"], b["cnt"], 2, 64, 4)
    lins = [blk["experts"][e][n] for e in sel for n in ("gate", "up")]
    outs = [torch.empty(1, m1.shape.inter, device=dev, dtype=torch.float16) for _ in lins]
    multi = lambda: ops.linear_fwd_multi(x, lins, outs)
    nb = 4 * m1.shape.inter * m1.shape.hidden * BPW
    lt = {"grouped_gate_up": [], "multi_gate_up": []}
    for fn in (grouped, multi):
        fn()
    for _ in range(args.rounds):
        lt["grouped_gate_up"].append(timed(dev, grouped, 50))
        lt["multi_gate_up"].append(timed(dev, multi, 50))
    res = {"experts": sel, "bytes": int(nb)}
    for k, v in lt.items():
        res[k + "_us"] = round(1000 * statistics.median(v), 2)
        res[k + "_gb_per_s"] = round(nb / statistics.median(v) / 1e6, 1)
    print(json.dumps({**res, **info}), flush=True)
    print(json.dumps({"clocks": sampler.stop(), **info}), flush=True)


if __name__ == "__main__":
    main()
