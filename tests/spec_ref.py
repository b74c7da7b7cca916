"""Host restatement of speculative decoding (include/hqq_b200.h, "Speculative decoding"): the prompt-lookup drafts, the greedy accept
rule, and a float64 reference with a per-element bound for the verify attention (hqq_b200_glue_attn_verify_split).

The bound is attn_split_ref's, applied per column: column (t, h) of slot b attends over cache rows 0 .. pos + t with the chunk
of the window end pos + n, so its tiles per warp, splits and roundings are those of a split-KV decode at that chunk."""
import math

import torch

import attn_split_ref as R


def ngram_drafts(hist, pos, tok, K):
    """hist: list of tokens (index p = the token fed at p, p < pos), tok at pos.  Returns K drafts."""
    seq = list(hist[:pos]) + [tok]
    L = len(seq)
    for g in (3, 2, 1):
        if L < g + 1:
            continue
        suf = seq[L - g:]
        js = [j for j in range(0, L - g) if seq[j:j + g] == suf]  # j + g <= L - 1
        if js:
            j = max(js)
            return [seq[j + g + i] if j + g + i < L else -1 for i in range(K)]
    return [-1] * K


def accept(tok, drafts, targets, pos, cache_len):
    """(emitted tokens, a, new pos).  targets: K + 1 greedy targets of the window rows."""
    K = len(drafts)
    n = min(K + 1, cache_len - pos)
    a = 0
    while a + 1 < n and drafts[a] == targets[a]:
        a += 1
    return list(drafts[:a]) + [targets[a]], a, (pos + a + 1) % cache_len


def verify_reference(q_rot, kc, vc, pos, T, dtype, S):
    """q_rot [B T, hq 128] (row b T + t), caches [B, hkv, L, 128] after the append.  Returns (y, bound) float64 [B T, hq 128]; rows
    t >= n[b] are NaN in y (their output means nothing) and inf in the bound."""
    B, hkv, L, HD = kc.shape
    hq = q_rot.shape[1] // HD
    G = hq // hkv
    u = 2.0 ** -(R.MANT[dtype] + 1)
    sl = R.LOG2E / math.sqrt(HD)
    y = torch.full((B * T, hq, HD), float("nan"), dtype=torch.float64, device=q_rot.device)
    bound = torch.full_like(y, float("inf"))
    for b in range(B):
        p = pos[b]
        n = min(T, L - p)
        end = p + n
        c = -(-end // S)
        chunk = -(-c // R.TILE) * R.TILE
        tiles_w = -(-(-(-chunk // R.TILE)) // R.NW)
        n_acc = tiles_w + R.NW + S + 4
        for t in range(n):
            for g in range(hkv):
                Q = q_rot[b * T + t].view(hq, HD)[g * G:(g + 1) * G].double()
                K = kc[b, g, :p + t + 1].double()
                V = vc[b, g, :p + t + 1].double()
                s = (Q @ K.T) / math.sqrt(HD)
                e = torch.exp(s - s.max(dim=1, keepdim=True).values)
                w = e / e.sum(1, keepdim=True)
                yy = w @ V
                A = w @ V.abs()
                dx = sl * 16 * 2.0 ** -23 * (Q.abs() @ K.abs().T) + 2.0 ** -22 * (s * math.sqrt(HD) * sl).abs()
                eta = u + math.log(2) * dx.max(dim=1, keepdim=True).values * 1.01 + (tiles_w + 6) * 2.0 ** -21
                E = (2 * eta / (1 - eta) + (2 * n_acc + 1) * 2.0 ** -23) * A * 1.01
                if dtype == torch.float16:
                    small = (e < 2.0 ** -13).double()
                    E = E + 2.0 ** -25 * ((small.unsqueeze(2) * (V.unsqueeze(0) - yy.unsqueeze(1)).abs()).sum(1)) / e.sum(1, keepdim=True)
                y[b * T + t, g * G:(g + 1) * G] = yy
                bound[b * T + t, g * G:(g + 1) * G] = E + 0.5 * R.ulp(yy.abs() + E, dtype)
    return y.view(B * T, hq * HD), bound.view(B * T, hq * HD)


def verify_defects(q_rot, kc, vc, pos, T):
    """Four defective outputs (float64, NaN where undefined): the mask off by one (column t sees pos + t + 1), the draft rows dropped
    (column t sees only <= pos), the column -> head mapping transposed (column (t, h) gets (h, t) where that exists), a dropped
    split (keys 0 .. 15 missing)."""
    B, hkv, L, HD = kc.shape
    hq = q_rot.shape[1] // HD
    G = hq // hkv
    outs = [torch.full((B * T, hq, HD), float("nan"), dtype=torch.float64, device=q_rot.device) for _ in range(4)]

    def att(Q, K, V):
        s = (Q @ K.T) / math.sqrt(HD)
        return torch.softmax(s, dim=-1) @ V

    for b in range(B):
        p = pos[b]
        n = min(T, L - p)
        for t in range(n):
            for g in range(hkv):
                Q = q_rot[b * T + t].view(hq, HD)[g * G:(g + 1) * G].double()
                kk, vv = kc[b, g].double(), vc[b, g].double()
                sl = slice(g * G, (g + 1) * G)
                if p + t + 2 <= L:
                    outs[0][b * T + t, sl] = att(Q, kk[:p + t + 2], vv[:p + t + 2])
                outs[1][b * T + t, sl] = att(Q, kk[:p + 1], vv[:p + 1])
                if p + t + 1 > 16:
                    outs[3][b * T + t, sl] = att(Q, kk[16:p + t + 1], vv[16:p + t + 1])
                for h in range(G):
                    if h < n and t < G:  # transposed: column (t, h) takes row h's query of head t, with row h's mask
                        outs[2][b * T + t, g * G + h] = att(q_rot[b * T + h].view(hq, HD)[g * G + t].double().view(1, HD), kk[:p + h + 1],
                                                            vv[:p + h + 1]).view(-1)
    return [o.view(B * T, hq * HD) for o in outs]
