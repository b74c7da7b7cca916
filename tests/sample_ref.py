"""Float64 restatement of hqq_b200_glue_sample (include/hqq_b200.h) for the tests: the kept set, the race, the rule that decides
when the kernel's fp32 arithmetic may pick another token than float64, and the planted defects.

Where the kernel may differ from float64:
  * the race: its key l / T + g is fp32.  l / T is rounded once (2^-24 relative), g = -log(-log u) carries the error of two
    logf calls (1 ulp each: about 2^-23 of t = -log u, which moves g by 2^-23, plus 2^-23 of g itself), and the sum is rounded once
    (2^-24 of the key).  KEY_REL and KEY_ABS bound that with a factor 4 of room; two kept elements whose float64 keys lie within the
    sum of their bounds may come out of the kernel in either order.
  * top-p: the masses are round(2^32 w) of the fp32 w = exp((l - max) / T): (l - max) / T rounds twice (2^-24 each, relative), expf
    is within 2 ulp, so w_i is within w_i (|x_i| 2^-23 + 2^-21) of exp(x_i), plus half a unit of 2^-32.  A distinct value whose
    cumulative share of the mass lies within that error (summed over the row, relative to the total) of top_p may sit on either
    side of the threshold."""
import math

import torch

KEY_REL = 2.0 ** -21
KEY_ABS = 2.0 ** -20


def fp32(x: float) -> float:
    return float(torch.tensor(float(x), dtype=torch.float32))


def keep_topk(lv, k, strict=False):
    n = lv.shape[-1]
    if not 0 < k < n:
        return torch.ones_like(lv, dtype=torch.bool)
    pivot = torch.topk(lv, k, dim=-1).values[:, -1:]
    return lv > pivot if strict else lv >= pivot


def masses(lv, keep, T):
    w = torch.where(keep, torch.exp((lv - lv.amax(dim=-1, keepdim=True)) / T), torch.zeros_like(lv))
    return w


def keep_topp(lv, keep, T, P):
    """Value threshold of top-p over `keep` (float64 masses)."""
    if P >= 1.0:
        return keep
    n = lv.shape[-1]
    w = masses(lv, keep, T)
    vs, order = torch.sort(torch.where(keep, lv, torch.full_like(lv, -math.inf)), dim=-1, descending=True)
    cum = w.gather(1, order).cumsum(dim=-1)
    j = (cum < P * cum[:, -1:]).sum(dim=-1, keepdim=True).clamp(max=n - 1)
    return keep & (lv >= vs.gather(1, j))


def race_keys(lv, T, u):
    return lv / T - torch.log(-torch.log(u))


def restate(logits, T, k, P, u, defect=None):
    """Tokens [rows] from logits [rows, n] (16-bit) and the uniforms u [rows, n] (philox_uniforms), with one planted defect:
    "temperature ignored", "strict pivot", "top-p before top-k"; the uniform defects are made by the caller on u."""
    T, P = fp32(T), fp32(P)
    lv = logits.double()
    Te = 1.0 if defect == "temperature ignored" else T
    if defect == "top-p before top-k":
        keep = keep_topp(lv, torch.ones_like(lv, dtype=torch.bool), Te, P) & keep_topk(lv, k)
    else:
        keep = keep_topp(lv, keep_topk(lv, k, strict=defect == "strict pivot"), Te, P)
    key = torch.where(keep, race_keys(lv, Te, u), torch.full_like(lv, -math.inf))
    return torch.argmax(key, dim=-1)


def accepted(logits, T, k, P, u):
    """Per row: (float64 token, the set of tokens the kernel may return, why the set has more than one: "" / "race" / "top-p")."""
    T, P = fp32(T), fp32(P)
    lv = logits.double()
    rows, n = lv.shape
    base = keep_topk(lv, k)
    key = race_keys(lv, T, u)
    err = KEY_REL * (lv.abs() / T + key.abs()) + KEY_ABS * ((key - lv / T).abs() + 1)
    out = []
    for b in range(rows):
        keeps = [keep_topp(lv[b:b + 1], base[b:b + 1], T, P)[0]]
        why = ""
        if P < 1.0:  # thresholds within the mass error of top_p
            w = masses(lv[b:b + 1], base[b:b + 1], T)[0]
            x = (lv[b] - lv[b].max()) / T
            tol = 2 * (float((w * (x.abs() * 2.0 ** -23 + 2.0 ** -21)).sum()) + n * 2.0 ** -33) / float(w.sum())
            vs, order = torch.sort(lv[b][base[b]], descending=True)
            cum = w[base[b]][order].cumsum(0)
            last = torch.ones_like(vs, dtype=torch.bool)
            last[:-1] = vs[:-1] != vs[1:]
            vals, share = vs[last].tolist(), (cum[last] / cum[-1]).tolist()  # distinct values, descending; mass share of l >= value
            for j, (v, s) in enumerate(zip(vals, share)):
                if abs(s - P) <= tol:  # v, or the next value up when v's share falls short
                    keeps.append(base[b] & (lv[b] >= v))
                    if j > 0:
                        keeps.append(base[b] & (lv[b] >= vals[j - 1]))
        tokens = set()
        for kp in keeps:
            kk = torch.where(kp, key[b], torch.full_like(key[b], -math.inf))
            win = int(torch.argmax(kk))
            near = kp & (kk >= kk[win] - err[b][win] - err[b])
            cand = set(int(i) for i in torch.nonzero(near).flatten().tolist())
            if len(cand) > 1:
                why = why or "race"
            tokens |= cand
        t0 = int(torch.argmax(torch.where(keeps[0], key[b], torch.full_like(key[b], -math.inf))))
        if len(keeps) > 1 and len(tokens) > 1 and not why:
            why = "top-p"
        out.append((t0, tokens, why))
    return out
