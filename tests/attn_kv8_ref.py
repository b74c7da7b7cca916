"""Test data and float64 reference for the split-KV decode attention over the 8-bit HQQ KV cache
(hqq_b200_glue_rope_attn_decode_split_kv8, csrc/decode_glue.cu).

The kernel attends to the dequantised cache rows with the arithmetic of hqq_b200_glue_rope_attn_decode_split, so the per-element
bound of tests/attn_split_ref.py holds against float64 softmax attention over those rows, row pos being
dequant(quant(rope(k))) and dequant(quant(v)).  `make_case` takes that module's case (its anchors make a dropped split visible) and
gives the fresh v row one outlier per group: quantising it then moves the small entries by up to a level (about 0.1), so a kernel
that attends to the raw row instead breaks the bound.  `defects` models four faults from the same data.

Everything is torch and runs on the tensors' device."""
import torch

import attn_split_ref as R
from hqq_b200.harness import kv8_dequantize, kv8_quantize_rows

HD = R.HD


def make_case(gen, batch, hq, hkv, cache_len, pos, dtype, cos, sin, gs, device):
    """R.make_case plus the 8-bit caches of its rows: levels kq / vq and meta ks, kz, vs, vz [batch, hkv, cache_len, .]."""
    case = R.make_case(gen, batch, hq, hkv, cache_len, pos, dtype, cos, sin, device)
    sign = torch.where(torch.arange(HD, device=device) % 2 == 0, 1.0, -1.0)
    fresh = 0.05 * sign
    fresh[::gs] = 60.0
    case["v"] = fresh.repeat(batch, hkv).to(dtype)
    for n in ("k", "v"):
        lv, sc, ze = kv8_quantize_rows(case[n + "c"], gs)
        case[n + "q"], case[n + "s"], case[n + "z"] = lv, sc, ze
    return case


def expected_caches(case, pos, cos, sin, gs):
    """The 8-bit caches after the call: row pos replaced by the quantised rope(k) and v, nothing else touched."""
    batch, hkv = case["kq"].shape[:2]
    out = {n: case[n].clone() for n in ("kq", "ks", "kz", "vq", "vs", "vz")}
    kr = R.rope(case["k"].view(batch, hkv, HD), cos[pos], sin[pos])
    for n, x in (("k", kr), ("v", case["v"].view(batch, hkv, HD))):
        lv, sc, ze = kv8_quantize_rows(x, gs)
        out[n + "q"][:, :, pos], out[n + "s"][:, :, pos], out[n + "z"][:, :, pos] = lv, sc, ze
    return out


def dequant(c, n, end):
    return kv8_dequantize(c[n + "q"][:, :, :end], c[n + "s"][:, :, :end], c[n + "z"][:, :, :end])


def reference(case, pos, cos, sin, S, dtype, gs):
    """y* [batch, hq * 128] in float64 over the dequantised caches, the bound of attn_split_ref (the same terms, computed over
    these rows), and the expected 8-bit caches."""
    import math
    exp = expected_caches(case, pos, cos, sin, gs)
    batch, hkv = exp["kq"].shape[:2]
    hq = case["q"].shape[1] // HD
    G = hq // hkv
    K, V = dequant(exp, "k", pos + 1).double(), dequant(exp, "v", pos + 1).double()
    qr = R.rope(case["q"].view(batch, hq, HD), cos[pos], sin[pos]).double()
    tiles_w = -(-(-(-R.chunk_len(pos, S) // R.TILE)) // R.NW)
    u = 2.0 ** -(R.MANT[dtype] + 1)
    sl = R.LOG2E / math.sqrt(HD)
    n_acc = tiles_w + R.NW + S + 4
    y = torch.empty(batch, hq, HD, dtype=torch.float64, device=qr.device)
    bound = torch.empty_like(y)
    for b in range(batch):
        for g in range(hkv):
            Q, Kg, Vg = qr[b, g * G:(g + 1) * G], K[b, g], V[b, g]
            yy, w, e, s = R._attend(Q, Kg, Vg)
            A = w @ Vg.abs()
            dx = sl * 16 * 2.0 ** -23 * (Q.abs() @ Kg.abs().T) + 2.0 ** -22 * (s * math.sqrt(HD) * sl).abs()
            eta = u + math.log(2) * dx.max(dim=1, keepdim=True).values * 1.01 + (tiles_w + 6) * 2.0 ** -21
            E = (2 * eta / (1 - eta) + (2 * n_acc + 1) * 2.0 ** -23) * A * 1.01
            if dtype == torch.float16:
                small = (e < 2.0 ** -13).double()
                E = E + 2.0 ** -25 * ((small.unsqueeze(2) * (Vg.unsqueeze(0) - yy.unsqueeze(1)).abs()).sum(1)) / e.sum(1, keepdim=True)
            y[b, g * G:(g + 1) * G] = yy
            bound[b, g * G:(g + 1) * G] = E + 0.5 * R.ulp(yy.abs() + E, dtype)
    return y.view(batch, hq * HD), bound.view(batch, hq * HD), exp


def attend(case, exp, pos, cos, sin, keep=None, k_rows=None, v_rows=None):
    """float64 attention of the rotated q over the given K / V rows [batch, hkv, pos + 1, 128] (default: the dequantised caches),
    optionally restricted to positions `keep`."""
    batch, hkv = exp["kq"].shape[:2]
    hq = case["q"].shape[1] // HD
    G = hq // hkv
    K = dequant(exp, "k", pos + 1).double() if k_rows is None else k_rows.double()
    V = dequant(exp, "v", pos + 1).double() if v_rows is None else v_rows.double()
    qr = R.rope(case["q"].view(batch, hq, HD), cos[pos], sin[pos]).double()
    out = torch.empty(batch, hq * HD, dtype=torch.float64, device=qr.device)
    for b in range(batch):
        for g in range(hkv):
            Kg, Vg = K[b, g], V[b, g]
            if keep is not None:
                Kg, Vg = Kg[keep], Vg[keep]
            out[b, g * G * HD:(g + 1) * G * HD] = R._attend(qr[b, g * G:(g + 1) * G], Kg, Vg)[0].reshape(-1)
    return out


def defects(case, exp, pos, cos, sin, S, gs):
    """Four faulty outputs from the same data: row pos attended unquantised; every row dequantised with the next group's scale;
    every zero one level off; split 0's partial dropped (pos >= 2)."""
    batch, hkv = exp["kq"].shape[:2]
    K, V = dequant(exp, "k", pos + 1), dequant(exp, "v", pos + 1)
    raw_k, raw_v = K.clone(), V.clone()
    raw_k[:, :, pos] = R.rope(case["k"].view(batch, hkv, HD), cos[pos], sin[pos])
    raw_v[:, :, pos] = case["v"].view(batch, hkv, HD)
    unquantised = attend(case, exp, pos, cos, sin, k_rows=raw_k, v_rows=raw_v)
    nb = {n: c.clone() for n, c in exp.items()}
    for n in ("ks", "vs"):
        flat = exp[n].reshape(batch, hkv, -1)
        nb[n] = flat.roll(-1, dims=2).reshape(exp[n].shape)
    neighbour = attend(case, nb, pos, cos, sin)
    off = {n: c.clone() for n, c in exp.items()}
    for n in ("kz", "vz"):
        off[n] = (exp[n].float() + 1.0).to(exp[n].dtype)
    zero_off = attend(case, off, pos, cos, sin)
    drop = min(R.chunk_len(pos, S), pos + 1)
    if drop <= pos:
        dropped = attend(case, exp, pos, cos, sin, keep=torch.arange(drop, pos + 1, device=K.device))
    else:
        dropped = torch.full_like(unquantised, float("nan"))
    return {"row pos unquantised": unquantised, "neighbouring group's scale": neighbour, "zero one level off": zero_off, "split 0 dropped": dropped}
