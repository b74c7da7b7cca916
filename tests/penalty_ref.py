"""fp32 restatement of hqq_b200_glue_penalize (include/hqq_b200.h) for the tests, written from the header's definition.

Row r of logits belongs to slot r // rows_per_slot.  A decode step first counts its token (counts[b][tok[b]] += 1 once per slot,
tok in [0, n)), then every element with c = counts, seen = c > 0 or prompt, x = fp32(l) becomes
    seen:  x = x * r if x < 0 else x / r
    c > 0: x = (x - f * c) - p
rounded once to the logits dtype; unseen elements keep their bits.  Every step is one torch fp32 operation (round to nearest, no
contraction), so the kernel's bits must come out."""
import torch


def count(counts, tok):
    """counts int32 [slots, n] after a step that consumes tok int64 [slots] (None: a prefill head, nothing counted)."""
    counts = counts.clone()
    if tok is not None:
        n = counts.shape[1]
        for b, t in enumerate(tok.tolist()):
            if 0 <= t < n:
                counts[b, t] += 1
    return counts


def penalize(logits, rows_per_slot, rep, freq, pres, counts, prompt, tok=None):
    """(penalised rows [rows, n] in the logits dtype, the counts after the step)."""
    counts = count(counts, tok)
    rows, n = logits.shape
    slot = torch.arange(rows) // rows_per_slot
    c = counts[slot]
    seen = (c > 0) | (prompt[slot] != 0)
    r, f, p = rep[slot].view(-1, 1), freq[slot].view(-1, 1), pres[slot].view(-1, 1)
    x = logits.float()
    y = torch.where(x < 0, torch.mul(x, r), torch.div(x, r))
    fc = torch.mul(f, c.to(torch.float32))
    y = torch.where(c > 0, torch.sub(torch.sub(y, fc), p), y)
    return torch.where(seen, y.to(logits.dtype), logits), counts
