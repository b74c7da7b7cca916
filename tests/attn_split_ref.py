"""Test data, float64 reference and per-element error bound for the split-KV decode attention
(hqq_b200_glue_rope_attn_decode_split, csrc/decode_glue.cu).

The kernel computes, for each query head h of kv group g at position pos,
    y = sum_t P_t v_t / sum_t P_t,     P_t = T(2^(x_t - m)) * (rescale factors),   x_t = fl(q_h . k_t) * fl(log2(e) / sqrt(d))
with the scores from mma.sync (fp32 accumulation), P rounded to T for the second MMA and the row sum adding the rounded P, then
fp32 merges across 8 warps and S splits and one rounding to T.  Every factor that multiplies P_t (the running max rescales, the
warp and split merges) multiplies the numerator and the denominator alike, so each P_t is perturbed by a relative eta_t and
    |y - y*| <= 2 eta / (1 - eta) * A  +  (2 n_acc + 1) 2^-23 A  +  sub  +  1/2 ulp_T(|y*| + ...)      A = sum_t w_t |v_t|
where y* = softmax(q k^T / sqrt(d)) v in float64 (w its weights) and
    eta   = u_T                                  rounding P to T (2^-11 fp16, 2^-8 bf16)
          + ln 2 * max_t dx_t * 1.01             score error in log2 units: dx_t = sl * 16 * 2^-23 * sum_i |q_i k_ti| + 2^-22 |x_t|
          + (n_tiles_per_warp + 6) * 2^-21       exp2f of every rescale factor and of P itself
    n_acc = n_tiles_per_warp + 8 + S + 4         fp32 additions into one output (MMA steps, warp merge, split merge, division)
    sub   = 2^-25 * sum_{t: e_t < 2^-13} |v_t - y*| / sum_t e_t   (fp16 only: P below the normal range is rounded absolutely; such
            a P is below 2^-14 of its warp's running max, hence e_t = exp(s_t - max s) < 2^-13)
2^-23 per MMA step, not 2^-24, allows for tensor-core accumulation that truncates (as tests/fused_ref.py does).

`make_case` plants three anchors so that the three defects `defects` models are each far outside that bound: cache row 0 and
row pos-1 and the fresh key at pos all point along the group's summed query, with logit ln(pos + 1) + 1 and distinct values.

Everything is torch and runs on the tensors' device."""
import math

import torch

MANT = {torch.float16: 10, torch.bfloat16: 7}
EMIN = {torch.float16: -14, torch.bfloat16: -126}
HD, TILE, NW = 128, 16, 8
LOG2E = 1.4426950408889634


def ulp(v, dtype):
    a = v.abs().to(torch.float64)
    e = torch.floor(torch.log2(torch.clamp(a, min=2.0 ** EMIN[dtype])))
    return torch.pow(2.0, e - MANT[dtype])


def split_count(sms, n_kv, cache_len):
    """S of the kernel: max(1, min(SMs / n_kv, ceil(cache_len / 16)))."""
    return max(1, min(sms // n_kv, -(-cache_len // TILE)))


def chunk_len(pos, S):
    """Positions per split at *pos: ceil((pos + 1) / S) rounded up to the 16-position tile."""
    c = -(-(pos + 1) // S)
    return -(-c // TILE) * TILE


def workspace_bytes(sms, hq, hkv, batch):
    return batch * hkv * max(1, sms // hkv) * (hq // hkv) * (HD + 2) * 4 + batch * hkv * 4


def tables(cache_len, dtype, device, theta=500000.0):
    inv = 1.0 / (theta ** (torch.arange(0, HD, 2, device=device, dtype=torch.float32) / HD))
    fr = torch.outer(torch.arange(cache_len, device=device, dtype=torch.float32), inv)
    return torch.cat([fr.cos(), fr.cos()], -1).to(dtype), torch.cat([fr.sin(), fr.sin()], -1).to(dtype)


def rope(x, cos, sin):
    """x*cos + rotate_half(x)*sin with each product and the sum rounded to T (the kernels' and the framework ops' rounding)."""
    dt, half = x.dtype, x.shape[-1] // 2
    rot = torch.cat([-x[..., half:], x[..., :half]], -1)
    a = (x.float() * cos.float()).to(dt).float()
    b = (rot.float() * sin.float()).to(dt).float()
    return (a + b).to(dt)


def make_case(gen, batch, hq, hkv, cache_len, pos, dtype, cos, sin, device):
    """Random q, k, v [batch, heads * 128] and caches [batch, hkv, cache_len, 128] in T, with the three anchors planted."""
    G = hq // hkv
    rn = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float32, device=device)  # gen lives on `device`
    q = rn(batch, hq * HD).to(dtype)
    k = rn(batch, hkv * HD).to(dtype)
    v = rn(batch, hkv * HD).to(dtype)
    kc = rn(batch, hkv, cache_len, HD).to(dtype)
    vc = rn(batch, hkv, cache_len, HD).to(dtype)
    c64, s64 = cos[pos].double(), sin[pos].double()
    qr = rope(q.view(batch, hq, HD), cos[pos], sin[pos]).double()
    lam = math.log(pos + 1) + 1.0
    sign = torch.where(torch.arange(HD, device=device) % 2 == 0, 1.0, -1.0).double()
    block = torch.where(torch.arange(HD, device=device) < HD // 2, 1.0, -1.0).double()
    for b in range(batch):
        for g in range(hkv):
            qg = qr[b, g * G:(g + 1) * G]
            u = qg.sum(0)
            u = u / u.norm()
            c = lam * math.sqrt(HD) / float((qg @ u).mean())
            anchor = (c * u).to(dtype)
            kc[b, g, 0] = anchor
            vc[b, g, 0] = (4.0 * sign).to(dtype)
            if pos >= 1:
                kc[b, g, pos - 1] = anchor
                vc[b, g, pos - 1] = (-4.0 * block).to(dtype)
            y = c * u  # the fresh key: the inverse rotation of c u, so that rope(k) points along u
            rot = torch.cat([-y[HD // 2:], y[:HD // 2]])
            k[b, g * HD:(g + 1) * HD] = (y * c64 - rot * s64).to(dtype)
            v[b, g * HD:(g + 1) * HD] = (3.0 * sign * block).to(dtype)
    return {"q": q, "k": k, "v": v, "kc": kc, "vc": vc}


def expected_caches(case, pos, cos, sin):
    """The caches after the call: row pos replaced by rope(k) and v, nothing else touched."""
    batch, hkv = case["kc"].shape[:2]
    kc, vc = case["kc"].clone(), case["vc"].clone()
    kc[:, :, pos] = rope(case["k"].view(batch, hkv, HD), cos[pos], sin[pos])
    vc[:, :, pos] = case["v"].view(batch, hkv, HD)
    return kc, vc


def _attend(Q, K, V):
    s = (Q @ K.T) / math.sqrt(HD)
    e = torch.exp(s - s.max(dim=1, keepdim=True).values)
    w = e / e.sum(1, keepdim=True)
    return w @ V, w, e, s


def reference(case, pos, cos, sin, S, dtype):
    """y* [batch, hq * 128] in float64 and the per-element bound of the module docstring; kc/vc the expected caches."""
    batch, hkv = case["kc"].shape[:2]
    hq = case["q"].shape[1] // HD
    G = hq // hkv
    kc, vc = expected_caches(case, pos, cos, sin)
    qr = rope(case["q"].view(batch, hq, HD), cos[pos], sin[pos]).double()
    chunk = chunk_len(pos, S)
    tiles_w = -(-(-(-chunk // TILE)) // NW)
    u = 2.0 ** -(MANT[dtype] + 1)
    sl = LOG2E / math.sqrt(HD)
    n_acc = tiles_w + NW + S + 4
    y = torch.empty(batch, hq, HD, dtype=torch.float64, device=qr.device)
    bound = torch.empty_like(y)
    for b in range(batch):
        for g in range(hkv):
            Q = qr[b, g * G:(g + 1) * G]
            K = kc[b, g, :pos + 1].double()
            V = vc[b, g, :pos + 1].double()
            yy, w, e, s = _attend(Q, K, V)
            A = w @ V.abs()
            dx = sl * 16 * 2.0 ** -23 * (Q.abs() @ K.abs().T) + 2.0 ** -22 * (s * math.sqrt(HD) * sl).abs()
            eta = u + math.log(2) * dx.max(dim=1, keepdim=True).values * 1.01 + (tiles_w + 6) * 2.0 ** -21
            E = (2 * eta / (1 - eta) + (2 * n_acc + 1) * 2.0 ** -23) * A * 1.01
            if dtype == torch.float16:
                small = (e < 2.0 ** -13).double()
                E = E + 2.0 ** -25 * ((small.unsqueeze(2) * (V.unsqueeze(0) - yy.unsqueeze(1)).abs()).sum(1)) / e.sum(1, keepdim=True)
            y[b, g * G:(g + 1) * G] = yy
            bound[b, g * G:(g + 1) * G] = E + 0.5 * ulp(yy.abs() + E, dtype)
    return y.view(batch, hq * HD), bound.view(batch, hq * HD), kc, vc


def defects(case, pos, cos, sin, S):
    """Three defective outputs from the same data: split 0's partial dropped; the stale cache row used at pos instead of the
    fresh key; position pos - 1 omitted.  (pos >= 2.)"""
    batch, hkv = case["kc"].shape[:2]
    hq = case["q"].shape[1] // HD
    G = hq // hkv
    kc, vc = expected_caches(case, pos, cos, sin)
    qr = rope(case["q"].view(batch, hq, HD), cos[pos], sin[pos]).double()
    drop = min(chunk_len(pos, S), pos + 1)
    outs = [torch.empty(batch, hq * HD, dtype=torch.float64, device=qr.device) for _ in range(3)]
    keep = torch.ones(pos + 1, dtype=torch.bool, device=qr.device)
    keep[pos - 1] = False
    for b in range(batch):
        for g in range(hkv):
            Q = qr[b, g * G:(g + 1) * G]
            K = kc[b, g, :pos + 1].double()
            V = vc[b, g, :pos + 1].double()
            sl = slice(g * G * HD, (g + 1) * G * HD)
            if drop <= pos:
                outs[0][b, sl] = _attend(Q, K[drop:], V[drop:])[0].reshape(-1)
            else:
                outs[0][b, sl] = float("nan")
            Ks = K.clone()
            Ks[pos] = case["kc"][b, g, pos].double()
            outs[1][b, sl] = _attend(Q, Ks, V)[0].reshape(-1)
            outs[2][b, sl] = _attend(Q, K[keep], V[keep])[0].reshape(-1)
    return outs


def within(out, y, bound):
    """(largest err / bound, all within)"""
    err = (out.double() - y).abs()
    ratio = err / bound
    ok = bool(torch.all(err <= bound))
    return float(torch.nan_to_num(ratio, nan=float("inf")).max()), ok
