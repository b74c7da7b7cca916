"""Sliding-window perplexity over a token stream with DecodeModel.score(), windowed as the reference's
examples/llama2_benchmark/eval_model.py::eval_wikitext2: windows of up to --max-length tokens every --stride tokens; window w's
loss is the mean negative log-likelihood of its last trg_len labels (the earlier ones are context), scaled by trg_len, and
perplexity = exp(sum of the windows' losses / end_loc).  The windows go as ragged slots, --batch of them per score() call.

DecodeModel builds random-weight models, so the number this prints measures the harness, not a language model: it says nothing about
how well any real checkpoint, quantised or not, models the text.

    python tools/perplexity.py [--tokens ids.pt | ids.npy] [--random 4096] [--vocab-limit 32000] [--max-length 1024] [--stride 512]
                               [--batch 8] [--shape 8b | tiny] [--layers 2] [--dtype fp16 | bf16] [--reference]"""
import argparse
import dataclasses
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@dataclasses.dataclass
class Window:
    begin: int    # tokens [begin, end) of the stream
    end: int
    trg_len: int  # eval_wikitext2's trg_len: labels before the window's last trg_len are context (-100)

    def scored(self):
        """[lo, hi) into score()'s entries for tokens[begin:end] (entry j predicts token begin + j + 1): the labels the loss keeps."""
        n = self.end - self.begin
        return max(n - self.trg_len, 1) - 1, n - 1


def windows(seq_len: int, max_length: int = 1024, stride: int = 512):
    """eval_wikitext2's loop: for i in range(0, seq_len, stride) the window [max(i + stride - max_length, 0), min(i + stride, seq_len))
    with trg_len = end - i.  Its perplexity divides by the last window's end."""
    out = []
    for i in range(0, seq_len, stride):
        end = min(i + stride, seq_len)
        out.append(Window(max(i + stride - max_length, 0), end, end - i))
    return out


def perplexity(wins, logprobs) -> float:
    """exp(sum over windows of trg_len * mean(-log p of the kept labels) / end_loc); logprobs[w] = score()'s entries for window w."""
    total = 0.0
    for w, lp in zip(wins, logprobs):
        lo, hi = w.scored()
        total += -float(lp[lo:hi].double().mean()) * w.trg_len
    return math.exp(total / wins[-1].end)


def score_windows(model, tokens, wins, batch):
    """score() of every window, `batch` windows per call as ragged slots starting at position 0; returns one fp32 tensor per window."""
    out = []
    for w0 in range(0, len(wins), batch):
        group = wins[w0:w0 + batch]
        prompts = [tokens[w.begin:w.end] for w in group] + [None] * (model.batch - len(group))
        lps = model.score(prompts)
        out += [lp.cpu() for lp in lps[:len(group)]]
    return out


def load_tokens(path):
    if path.endswith(".npy"):
        import numpy as np
        return torch.from_numpy(np.load(path)).flatten().to(torch.long)
    t = torch.load(path, map_location="cpu")
    if isinstance(t, dict):
        t = t["input_ids"]
    return torch.as_tensor(t).flatten().to(torch.long)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", help=".pt / .npy token ids (a tensor, or a dict with 'input_ids')")
    ap.add_argument("--random", type=int, default=4096, help="without --tokens: this many seeded random tokens")
    ap.add_argument("--vocab-limit", type=int, default=32000, help="random tokens are drawn from [0, vocab-limit)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-length", type=int, default=1024)
    ap.add_argument("--stride", type=int, default=512)
    ap.add_argument("--batch", type=int, default=8, help="windows per score() call")
    ap.add_argument("--shape", choices=["8b", "tiny"], default="8b")
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--dtype", choices=["fp16", "bf16"], default="fp16")
    ap.add_argument("--chunk", type=int, default=2048)
    ap.add_argument("--reference", action="store_true", help="fused=False: framework ops, the correctness reference")
    a = ap.parse_args()
    from hqq_b200 import harness
    if not torch.cuda.is_available():
        sys.exit("perplexity.py runs DecodeModel on a CUDA device")
    shape = harness.LLAMA3_8B if a.shape == "8b" else harness.TINY
    if a.tokens:
        tokens = load_tokens(a.tokens)
    else:
        g = torch.Generator().manual_seed(a.seed)
        tokens = torch.randint(0, min(a.vocab_limit, shape.vocab), (a.random,), generator=g)
    if int(tokens.min()) < 0 or int(tokens.max()) >= shape.vocab:
        sys.exit(f"token ids must lie in [0, {shape.vocab})")
    if tokens.numel() < 2:
        sys.exit("need at least two tokens")
    dev = torch.device("cuda")
    wins = windows(tokens.numel(), a.max_length, a.stride)
    batch = min(a.batch, len(wins))
    model = harness.DecodeModel(shape, dtype=torch.float16 if a.dtype == "fp16" else torch.bfloat16, device=dev, n_layers=a.layers,
                                cache_len=-(-a.max_length // 64) * 64, batch=batch, ragged=True, fused=False if a.reference else True)
    lps = score_windows(model, tokens.to(dev), wins, batch)
    print(json.dumps({"perplexity": perplexity(wins, lps), "tokens": int(tokens.numel()), "windows": len(wins), "max_length": a.max_length,
                      "stride": a.stride, "fused": not a.reference, "shape": a.shape, "layers": a.layers, "dtype": a.dtype,
                      "note": "random-weight model: not the perplexity of any real model"}))


if __name__ == "__main__":
    main()
