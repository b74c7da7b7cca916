"""Restatements of the mixture-of-experts glue (csrc/decode_glue.cu: hqq_b200_glue_moe_route / _combine) for the CPU and GPU tests.

route():   the router logits exactly in float64, rounded once to the model dtype (the kernel sums in fp32 and rounds once; transformers'
           MixtralTopKRouter computes F.linear in the model dtype), softmax in fp32, top-k with ties to the lower expert index, the k
           weights renormalised in fp32.
group():   the expert-major grouping the router also writes, from a given [M, k] id table: per-expert offset and count, the token of
           every slot, and the slot of every (token, j) pair -- ascending token order within an expert.
combine(): transformers 5.5 MixtralExperts.forward, experts visited in ascending order: (y * w) in fp32, .to(dtype), index_add_ into
           a zero tensor of the model dtype, one expert at a time."""
import torch

from fused_ref import round_to


def logits(x, router):
    """T(x @ router^T) with the exact product rounded once to T."""
    return round_to(x.to(torch.float64) @ router.to(torch.float64).T, x.dtype)


def route(x, router, k):
    """(ids int32 [M, k], weights fp32 [M, k], probabilities fp32 [M, E]) in the kernel's slot order (descending probability)."""
    p = torch.softmax(logits(x, router).float(), dim=-1)
    order = torch.sort(-p, dim=-1, stable=True).indices[:, :k]  # stable: equal probabilities keep the lower index first
    top = p.gather(1, order)
    return order.to(torch.int32), top / top.sum(dim=-1, keepdim=True), p


def group(ids, E):
    """(off [E], cnt [E], token [M k], pair_of [M, k]) as int32 for the id table ids [M, k]."""
    M, k = ids.shape
    ids = ids.long()
    cnt = torch.bincount(ids.reshape(-1), minlength=E)
    off = torch.cumsum(cnt, 0) - cnt
    token = torch.empty(M * k, dtype=torch.int32)
    pair_of = torch.empty(M, k, dtype=torch.int32)
    nxt = off.clone()
    for t in range(M):
        for j in range(k):
            e = int(ids[t, j])
            token[nxt[e]] = t
            pair_of[t, j] = int(nxt[e])
            nxt[e] += 1
    return off.to(torch.int32), cnt.to(torch.int32), token, pair_of


def combine(y, ids, weights, pair_of, E):
    """delta [M, H] in y's dtype from the slot-ordered expert outputs y [M k, H]."""
    M = ids.shape[0]
    dt = y.dtype
    out = torch.zeros(M, y.shape[1], dtype=dt, device=y.device)
    for e in range(E):
        t, j = (ids.long() == e).nonzero(as_tuple=True)
        if t.numel() == 0:
            continue
        term = (y[pair_of.long()[t, j]].float() * weights[t, j, None].float()).to(dt)
        out[t] = (out[t].float() + term.float()).to(dt)  # index_add_: one add per token and expert, rounded to dt
    return out


def near_tie(p, k, rel=1e-3):
    """Rows where two of the k + 1 largest probabilities are so close (but not equal) that a last-bit difference in a logit may
    swap them: the selection or the slot order of such a row may legitimately differ."""
    s = torch.sort(p, dim=-1, descending=True).values[:, :k + 1]
    gap = s[:, :-1] - s[:, 1:]
    return ((gap > 0) & (gap <= rel * s[:, :-1])).any(dim=1)
