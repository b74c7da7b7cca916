"""Test data and float64 reference for the split-KV decode attention over the 4-bit HQQ KV cache
(hqq_b200_glue_rope_attn_decode_split_kv4, csrc/decode_glue.cu).

The 8-bit reference (tests/attn_kv8_ref.py) carries over: the kernel attends to the dequantised rows with the arithmetic of the
16-bit split kernel, so the bound of tests/attn_split_ref.py holds against float64 attention over those rows, row pos being
dequant(quant(rope(k))) and dequant(quant(v)).  Only the format differs: levels are packed two to a byte
(kv8_quantize_rows(..., bits=4)), and the planted faults include the one a 4-bit kernel can make, high and low nibble swapped.

Everything is torch and runs on the tensors' device."""
import math

import torch

import attn_split_ref as R
from hqq_b200.harness import kv8_dequantize, kv8_quantize_rows

HD = R.HD


def make_case(gen, batch, hq, hkv, cache_len, pos, dtype, cos, sin, gs, device):
    """R.make_case plus the 4-bit caches of its rows: packed levels kq / vq [batch, hkv, cache_len, 64] and meta ks, kz, vs, vz
    [batch, hkv, cache_len, 128 / gs].  The fresh v row has one outlier per group (a level is then about 4), so that quantising it
    moves the entries of +0.05 to -0.05 and a kernel that attends to the raw row breaks the bound."""
    case = R.make_case(gen, batch, hq, hkv, cache_len, pos, dtype, cos, sin, device)
    sign = torch.where(torch.arange(HD, device=device) % 2 == 0, 1.0, -1.0)
    fresh = 0.05 * sign
    fresh[::gs] = 60.0
    case["v"] = fresh.repeat(batch, hkv).to(dtype)
    for n in ("k", "v"):
        case[n + "q"], case[n + "s"], case[n + "z"] = kv8_quantize_rows(case[n + "c"], gs, 4)
    return case


def expected_caches(case, pos, cos, sin, gs):
    """The 4-bit caches after the call: row pos replaced by the quantised rope(k) and v, nothing else touched."""
    batch, hkv = case["kq"].shape[:2]
    out = {n: case[n].clone() for n in ("kq", "ks", "kz", "vq", "vs", "vz")}
    kr = R.rope(case["k"].view(batch, hkv, HD), cos[pos], sin[pos])
    for n, x in (("k", kr), ("v", case["v"].view(batch, hkv, HD))):
        lv, sc, ze = kv8_quantize_rows(x, gs, 4)
        out[n + "q"][:, :, pos], out[n + "s"][:, :, pos], out[n + "z"][:, :, pos] = lv, sc, ze
    return out


def dequant(c, n, end):
    return kv8_dequantize(c[n + "q"][:, :, :end], c[n + "s"][:, :, :end], c[n + "z"][:, :, :end], 4)


def reference(case, pos, cos, sin, S, dtype, gs):
    """y* [batch, hq * 128] in float64 over the dequantised caches, the bound of attn_kv8_ref.reference (the same terms over these
    rows), and the expected 4-bit caches."""
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
    """float64 attention of the rotated q over the given K / V rows (default: the dequantised caches), optionally restricted to
    positions `keep`."""
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
    """Five faulty outputs from the same data: high and low nibble swapped; every row dequantised with the next group's scale;
    every zero one level off; split 0's partial dropped (pos >= 2); row pos attended unquantised."""
    batch, hkv = exp["kq"].shape[:2]
    out = {}
    sw = dict(exp)
    for n in ("kq", "vq"):
        sw[n] = (exp[n] >> 4) | (exp[n] << 4)
    out["nibbles swapped"] = attend(case, sw, pos, cos, sin)
    nb = dict(exp)
    for n in ("ks", "vs"):
        nb[n] = exp[n].reshape(batch, hkv, -1).roll(-1, dims=2).reshape(exp[n].shape)
    out["neighbouring group's scale"] = attend(case, nb, pos, cos, sin)
    off = dict(exp)
    for n in ("kz", "vz"):
        off[n] = (exp[n].float() + 1.0).to(exp[n].dtype)
    out["zero one level off"] = attend(case, off, pos, cos, sin)
    drop = min(R.chunk_len(pos, S), pos + 1)
    if drop <= pos:
        out["split 0 dropped"] = attend(case, exp, pos, cos, sin, keep=torch.arange(drop, pos + 1, device=exp["kq"].device))
    K, V = dequant(exp, "k", pos + 1), dequant(exp, "v", pos + 1)
    K[:, :, pos] = R.rope(case["k"].view(batch, hkv, HD), cos[pos], sin[pos])
    V[:, :, pos] = case["v"].view(batch, hkv, HD)
    out["row pos unquantised"] = attend(case, exp, pos, cos, sin, k_rows=K, v_rows=V)
    return out
