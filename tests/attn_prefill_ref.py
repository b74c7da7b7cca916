"""Test data, float64 reference and per-element error bound for prompt prefill (hqq_b200_glue_rope_append_rows and
hqq_b200_glue_attn_prefill, csrc/decode_glue.cu).

Query t of a chunk sits at position p = pos0 + t.  For each of its heads the attention kernel computes
    y = sum_{j<=p} P_j v_j / sum_{j<=p} P_j,     P_j = T(2^(x_j - m)) * (rescale factors),   x_j = fl(q . k_j) * fl(log2(e) / sqrt(d))
with the scores from mma.sync (fp32 accumulation), key tiles of 64 positions taken in order from position 0, an online softmax
whose rescale factors and P come from exp2f, P rounded to T for the second MMA and the row sum adding the rounded P, then one
division and one rounding to T.  The argument of attn_split_ref carries over without the split merge:
    |y - y*| <= 2 eta / (1 - eta) * A  +  (2 n_acc + 1) 2^-23 A  +  sub  +  1/2 ulp_T(|y*| + ...)      A = sum_j w_j |v_j|
    eta   = u_T + ln 2 * max_j dx_j * 1.01 + (n_t + 6) * 2^-21      n_t = ceil((p + 1) / 64) tiles, one rescale each
    n_acc = 4 n_t + n_t + 4                                           MMA steps of 16 positions, rescale products, quad sum, division
dx_j is the score error of attn_split_ref (the score MMA is the same 8 steps of 16 dimensions).  sub (fp16 only, P below the
normal range) is attn_split_ref's term with |v_j - y*| <= |v_j| + |y*|, which keeps it a matrix product at 131072 positions.

`make_case` plants anchors for the chunk's last query t* (position p*) in every kv group g: cache rows 0, p* and p* + 1 point
along the group's summed query with logit ln(p* + 1) + 1 and carry distinct values whose sign alternates with g.  Each defect
`defects` models then moves that row far outside the bound: a causal mask off by one (rows see p + 1), the diagonal key
omitted, key tile 0 dropped, and (n_kv >= 2) the query heads of group g reading kv head g + 1.

Everything is torch and runs on the tensors' device."""
import math

import torch

from attn_split_ref import HD, LOG2E, MANT, rope, tables, ulp  # noqa: F401  (tables: re-exported for the tests)

KT = 64  # key positions per tile


def make_case(gen, batch, hq, hkv, cache_len, pos0, T, dtype, device):
    """Rotated queries q [batch*T, hq*128] (row b*T + t), caches [batch, hkv, cache_len, 128] in T, anchors planted (needs
    pos0 + T <= cache_len; the p* + 1 anchor only when pos0 + T < cache_len)."""
    G = hq // hkv
    rn = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float32, device=device)  # gen lives on `device`
    q = rn(batch * T, hq * HD).to(dtype)
    kc = rn(batch, hkv, cache_len, HD).to(dtype)
    vc = rn(batch, hkv, cache_len, HD).to(dtype)
    ps = pos0 + T - 1
    lam = math.log(ps + 1) + 1.0
    sign = torch.where(torch.arange(HD, device=device) % 2 == 0, 1.0, -1.0).double()
    block = torch.where(torch.arange(HD, device=device) < HD // 2, 1.0, -1.0).double()
    for b in range(batch):
        for g in range(hkv):
            qg = q[b * T + T - 1].view(hq, HD)[g * G:(g + 1) * G].double()
            u = qg.sum(0)
            u = u / u.norm()
            c = lam * math.sqrt(HD) / float((qg @ u).mean())
            anchor = (c * u).to(dtype)
            flip = -1.0 if g % 2 else 1.0
            kc[b, g, 0] = anchor
            vc[b, g, 0] = (4.0 * flip * sign).to(dtype)
            if ps >= 1:
                kc[b, g, ps] = anchor
                vc[b, g, ps] = (-4.0 * flip * block).to(dtype)
            if ps + 1 < cache_len:
                kc[b, g, ps + 1] = anchor
                vc[b, g, ps + 1] = (3.0 * flip * sign * block).to(dtype)
    return {"q": q, "kc": kc, "vc": vc}


def make_append_case(gen, batch, hq, hkv, cache_len, T, dtype, device):
    """Unrotated q [batch*T, hq*128], k / v [batch*T, hkv*128] and caches [batch, hkv, cache_len, 128] in T."""
    rn = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float32, device=device)
    return {"q": rn(batch * T, hq * HD).to(dtype), "k": rn(batch * T, hkv * HD).to(dtype), "v": rn(batch * T, hkv * HD).to(dtype),
            "kc": rn(batch, hkv, cache_len, HD).to(dtype), "vc": rn(batch, hkv, cache_len, HD).to(dtype)}


def expected_append(case, pos0, T, cos, sin):
    """(q_out, k_cache, v_cache) after hqq_b200_glue_rope_append_rows: rows [pos0, pos0 + T) replaced, nothing else touched."""
    batch, hkv = case["kc"].shape[:2]
    hq = case["q"].shape[1] // HD
    c, s = cos[pos0:pos0 + T].view(1, T, 1, HD), sin[pos0:pos0 + T].view(1, T, 1, HD)
    qo = rope(case["q"].view(batch, T, hq, HD), c, s).view(batch * T, hq * HD)
    kc, vc = case["kc"].clone(), case["vc"].clone()
    kc[:, :, pos0:pos0 + T] = rope(case["k"].view(batch, T, hkv, HD), c, s).transpose(1, 2)
    vc[:, :, pos0:pos0 + T] = case["v"].view(batch, T, hkv, HD).transpose(1, 2)
    return qo, kc, vc


def _masked(mode, j, p):
    """Keys row p sees: the kernel's j <= p, or one of the modelled defects."""
    if mode == "off by one":
        return j <= p + 1
    if mode == "diagonal omitted":
        return j < p
    if mode == "tile 0 dropped":
        return (j <= p) & (j >= KT)
    return j <= p


def _attend(case, pos0, T, dtype, mode="exact", with_bound=False):
    kc, vc = case["kc"], case["vc"]
    batch, hkv, L = kc.shape[:3]
    hq = case["q"].shape[1] // HD
    G = hq // hkv
    n_keys = min(pos0 + T + (1 if mode == "off by one" else 0), L)
    dev = kc.device
    u = 2.0 ** -(MANT[dtype] + 1)
    sl = LOG2E / math.sqrt(HD)
    y = torch.empty(batch * T, hq * HD, dtype=torch.float64, device=dev)
    bound = torch.empty_like(y) if with_bound else None
    tb = max(1, (1 << 22) // (G * n_keys))  # query positions per block: bounds the float64 temporaries
    j = torch.arange(n_keys, device=dev)
    for b in range(batch):
        for g in range(hkv):
            gk = (g + 1) % hkv if mode == "wrong kv head" else g
            K = kc[b, gk, :n_keys].double()
            V = vc[b, gk, :n_keys].double()
            for t0 in range(0, T, tb):
                t1 = min(T, t0 + tb)
                Q = case["q"][b * T + t0:b * T + t1].view(t1 - t0, hq, HD)[:, g * G:(g + 1) * G].reshape(-1, HD).double()
                p = (pos0 + torch.arange(t0, t1, device=dev)).repeat_interleave(G)  # row (t, h) -> position
                keep = _masked(mode, j.view(1, -1), p.view(-1, 1))
                s = (Q @ K.T) / math.sqrt(HD)
                s = s.masked_fill(~keep, -math.inf)
                e = torch.exp(s - s.max(dim=1, keepdim=True).values)
                w = e / e.sum(1, keepdim=True)
                yy = w @ V
                rows = slice(b * T + t0, b * T + t1)
                cols = slice(g * G * HD, (g + 1) * G * HD)
                y[rows, cols] = yy.view(t1 - t0, G * HD)
                if not with_bound:
                    continue
                A = w @ V.abs()
                x = (s * math.sqrt(HD) * sl).abs()
                dx = sl * 16 * 2.0 ** -23 * (Q.abs() @ K.abs().T) + 2.0 ** -22 * x.masked_fill(~keep, 0.0)
                dx = dx.masked_fill(~keep, 0.0)
                n_t = (p // KT + 1).double().view(-1, 1)
                eta = u + math.log(2) * dx.max(dim=1, keepdim=True).values * 1.01 + (n_t + 6) * 2.0 ** -21
                n_acc = 5 * n_t + 4
                E = (2 * eta / (1 - eta) + (2 * n_acc + 1) * 2.0 ** -23) * A * 1.01
                if dtype == torch.float16:
                    small = ((e < 2.0 ** -13) & keep).double()
                    E = E + 2.0 ** -25 * (small @ V.abs() + yy.abs() * small.sum(1, keepdim=True)) / e.sum(1, keepdim=True)
                bound[rows, cols] = (E + 0.5 * ulp(yy.abs() + E, dtype)).view(t1 - t0, G * HD)
    return y, bound


def reference(case, pos0, T, dtype):
    """y* [batch*T, hq*128] in float64 and the per-element bound of the module docstring."""
    return _attend(case, pos0, T, dtype, with_bound=True)


DEFECTS = ("off by one", "diagonal omitted", "tile 0 dropped", "wrong kv head")


def defects(case, pos0, T, dtype):
    """{defect name: defective output} from the same data (the wrong kv head only when n_kv >= 2, off by one only when the
    cache has a row past the chunk)."""
    hkv, L = case["kc"].shape[1], case["kc"].shape[2]
    out = {}
    for mode in DEFECTS:
        if (mode == "wrong kv head" and hkv < 2) or (mode == "off by one" and pos0 + T >= L):
            continue
        out[mode] = _attend(case, pos0, T, dtype, mode)[0]
    return out


def within(out, y, bound):
    """(largest err / bound, all within)"""
    err = (out.double() - y).abs()
    ratio = err / bound
    ok = bool(torch.all(err <= bound))
    return float(torch.nan_to_num(ratio, nan=float("inf")).max()), ok
