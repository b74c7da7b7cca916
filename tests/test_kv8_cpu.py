"""The 8-bit HQQ KV cache on the CPU kernel emulator: hqq_b200_glue_rope_attn_decode_split_kv8 and
hqq_b200_glue_rope_append_rows_kv8 (csrc/decode_glue.cu), and the framework-op format functions of the decode harness.

The emulator has 4 SMs, so S = max(1, min(4 / n_kv, ceil(cache_len / 16))).  Outputs are held to the per-element bound of
tests/attn_split_ref.py against float64 attention over the dequantised cache (tests/attn_kv8_ref.py); cache rows to HQQ's
Quantizer.quantize(row, nbits=8, axis=1, optimize=False) as the CPU oracle computes it, bit for bit."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import attn_kv8_ref as K8  # noqa: E402
import attn_split_ref as R  # noqa: E402
from hqq_b200.harness import kv8_dequantize, kv8_quantize_rows  # noqa: E402
from oracle import hqq_oracle as O  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
ONAME = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
SMS = 4
E_INVALID, E_UNSUPPORTED = -1, -2
VP, I = ctypes.c_void_p, ctypes.c_int


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_glue_rope_attn_decode_split_kv8.argtypes = [VP] * 14 + [I] * 7 + [VP]
    lib.hqq_b200_glue_rope_append_rows_kv8.argtypes = [VP] * 14 + [I] * 9 + [VP]
    lib.hqq_b200_glue_rope_append_rows.argtypes = [VP] * 8 + [I] * 8 + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def run_kv8(emu, case, pos, cos, sin, hq, hkv, dtype, gs, ws=None):
    batch, L = case["kq"].shape[0], case["kq"].shape[2]
    c = {n: case[n].clone() for n in ("kq", "ks", "kz", "vq", "vs", "vz")}
    out = torch.zeros(batch, hq * R.HD, dtype=dtype)
    if ws is None:
        ws = torch.zeros(R.workspace_bytes(SMS, hq, hkv, batch), dtype=torch.uint8)
    p = torch.tensor([pos], dtype=torch.int64)
    rc = emu.hqq_b200_glue_rope_attn_decode_split_kv8(P(case["q"]), P(case["k"]), P(case["v"]), P(cos), P(sin), P(c["kq"]), P(c["ks"]), P(c["kz"]),
                                                     P(c["vq"]), P(c["vs"]), P(c["vz"]), P(p), P(out), P(ws), hq, hkv, L, R.HD, gs, batch, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, c, ws


def oracle_rows(x, gs, dtype):
    """oracle.quantize of each row (float32 of the T values): levels uint8, scale and zero cast to T."""
    rows = x.reshape(-1, R.HD).float().numpy()
    lv, sc, ze = [], [], []
    for r in rows:
        W_q, meta = O.quantize(r.reshape(1, -1), nbits=8, group_size=gs, axis=1, optimize=False, bitpack=False)
        lv.append(np.asarray(W_q).reshape(-1).astype(np.uint8))
        sc.append(np.asarray(meta["scale"]).reshape(-1))
        ze.append(np.asarray(meta["zero"]).reshape(-1))
    shape = x.shape[:-1]
    ng = R.HD // gs
    return (torch.from_numpy(np.stack(lv)).reshape(shape + (R.HD,)), torch.from_numpy(np.stack(sc)).to(dtype).reshape(shape + (ng,)),
            torch.from_numpy(np.stack(ze)).to(dtype).reshape(shape + (ng,)))


def oracle_dequant(lv, scale, zero, gs, dtype):
    """oracle.dequantize of 8-bit levels with the meta in T: float32 values of T, shape [groups, gs]."""
    meta = {"packing": None, "zero": zero.float().reshape(-1, 1).numpy(), "scale": scale.float().reshape(-1, 1).numpy(), "nbits": 8,
            "shape": (lv.numel() // gs, gs)}
    deq = O.dequantize(lv.reshape(-1, gs).numpy().astype(np.float32), meta, ONAME[dtype])
    return torch.from_numpy(np.asarray(deq, dtype=np.float32))


def positions(L, S):
    c = R.TILE * max(1, (L // (2 * S)) // R.TILE)  # a chunk length whose S-fold fits the cache twice
    return sorted({0, 15, 16, 17, S * c - 1, S * c, S * c + 1, L - 1})


CASES = [(hq, hkv, B) for (hq, hkv) in ((2, 2), (8, 2), (8, 1)) for B in (1, 3)]


@pytest.mark.parametrize("gs", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv,B", CASES)
def test_emulated_kv8_attention_within_bound_and_row_pos_exact(emu, dtype, gs, hq, hkv, B):
    """Output within the bound over the dequantised cache (row pos = dequant(quant(rope(k)))) at tile and chunk edges; the row
    written at pos equals the oracle bit for bit and no other row changes; tickets back at zero; the four defects break the bound."""
    L = 300
    S = R.split_count(SMS, hkv, L)
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(1000 * hq + 100 * hkv + 10 * B + gs)
    for pos in positions(L, S):
        case = K8.make_case(gen, B, hq, hkv, L, pos, dtype, cos, sin, gs, "cpu")
        out, c, ws = run_kv8(emu, case, pos, cos, sin, hq, hkv, dtype, gs)
        y, bound, exp = K8.reference(case, pos, cos, sin, S, dtype, gs)
        for n in exp:
            assert torch.equal(c[n], exp[n]), (pos, n)
        kr = R.rope(case["k"].view(B, hkv, R.HD), cos[pos], sin[pos])
        for n, x in (("k", kr), ("v", case["v"].view(B, hkv, R.HD))):
            lv, sc, ze = oracle_rows(x, gs, dtype)
            assert torch.equal(c[n + "q"][:, :, pos], lv) and torch.equal(c[n + "s"][:, :, pos], sc) and torch.equal(c[n + "z"][:, :, pos], ze), (pos, n)
        assert torch.count_nonzero(ws[-4 * B * hkv:]) == 0, pos
        ratio, ok = R.within(out, y, bound)
        assert ok, (pos, ratio)
        if pos >= 2:
            for name, bad in K8.defects(case, exp, pos, cos, sin, S, gs).items():
                if name == "split 0 dropped" and S == 1:
                    continue
                assert not R.within(bad, y, bound)[1], (pos, name)


@pytest.mark.parametrize("gs", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_kv8_rows_kernel_matches_decode_rows_oracle_and_q(emu, dtype, gs):
    """The rows kernel writes the cache rows the decode kernel writes from the same k and v, stages oracle.dequantize of them, leaves
    every other row alone, and its q_out equals hqq_b200_glue_rope_append_rows' bit for bit."""
    hq, hkv, B, L, T, pos0 = 8, 2, 3, 96, 20, 33
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(gs + CODE[dtype])
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    q, k, v = rn(B * T, hq * R.HD), rn(B * T, hkv * R.HD), rn(B * T, hkv * R.HD)
    ng = R.HD // gs
    kq, vq = torch.randint(0, 256, (B, hkv, L, R.HD), generator=gen, dtype=torch.uint8), torch.randint(0, 256, (B, hkv, L, R.HD), generator=gen, dtype=torch.uint8)
    meta = [rn(B, hkv, L, ng) for _ in range(4)]
    kst, vst = rn(B, hkv, L, R.HD), rn(B, hkv, L, R.HD)
    c = [kq.clone(), meta[0].clone(), meta[1].clone(), vq.clone(), meta[2].clone(), meta[3].clone()]
    st = [kst.clone(), vst.clone()]
    qo = torch.zeros(B * T, hq * R.HD, dtype=dtype)
    rc = emu.hqq_b200_glue_rope_append_rows_kv8(P(q), P(k), P(v), P(cos), P(sin), *[P(t) for t in c], P(st[0]), P(st[1]), P(qo), pos0, T, hq, hkv, L,
                                                R.HD, gs, B, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    # q_out and the fp16 kernel's rows
    qx, kx, vx = torch.zeros_like(qo), torch.zeros(B, hkv, L, R.HD, dtype=dtype), torch.zeros(B, hkv, L, R.HD, dtype=dtype)
    assert emu.hqq_b200_glue_rope_append_rows(P(q), P(k), P(v), P(cos), P(sin), P(kx), P(vx), P(qx), pos0, T, hq, hkv, L, R.HD, B, CODE[dtype], None) == 0
    assert torch.equal(qo, qx)
    rows = slice(pos0, pos0 + T)
    outside = torch.ones(L, dtype=torch.bool)
    outside[rows] = False
    for (lvl, sc, ze, stg), (lvl0, sc0, ze0, stg0), x in (((c[0], c[1], c[2], st[0]), (kq, meta[0], meta[1], kst), kx),
                                                          ((c[3], c[4], c[5], st[1]), (vq, meta[2], meta[3], vst), vx)):
        ol, os_, oz = oracle_rows(x[:, :, rows], gs, dtype)
        assert torch.equal(lvl[:, :, rows], ol) and torch.equal(sc[:, :, rows], os_) and torch.equal(ze[:, :, rows], oz)
        for got, before in ((lvl, lvl0), (sc, sc0), (ze, ze0), (stg, stg0)):
            assert torch.equal(got[:, :, outside], before[:, :, outside])
        assert torch.equal(stg[:, :, rows].float(), oracle_dequant(ol, os_, oz, gs, dtype).reshape(stg[:, :, rows].shape))
    # the decode kernel's row at each position of the chunk from the same k and v
    for t in (0, T - 1):
        p = pos0 + t
        case = {"q": q.view(B, T, -1)[:, t].contiguous(), "k": k.view(B, T, -1)[:, t].contiguous(), "v": v.view(B, T, -1)[:, t].contiguous(),
                "kq": kq, "ks": meta[0], "kz": meta[1], "vq": vq, "vs": meta[2], "vz": meta[3]}
        _, d, _ = run_kv8(emu, case, p, cos, sin, hq, hkv, dtype, gs)
        for n, got in zip(("kq", "ks", "kz", "vq", "vs", "vz"), c):
            assert torch.equal(d[n][:, :, p], got[:, :, p]), (t, n)


@pytest.mark.parametrize("gs", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
def test_kv8_quantize_rows_equals_oracle(dtype, gs):
    """kv8_quantize_rows on random rows and rows of large magnitude equals oracle.quantize(..., nbits=8, axis=1, optimize=False) with
    the meta cast to T; kv8_dequantize equals oracle.dequantize."""
    gen = torch.Generator().manual_seed(gs)
    x = torch.cat([torch.randn(64, R.HD, generator=gen), torch.randn(16, R.HD, generator=gen).clamp(-6, 6) * 1e4, torch.randn(16, R.HD, generator=gen) * 1e-3])
    x = x.to(dtype)
    lv, sc, ze = kv8_quantize_rows(x, gs)
    ol, os_, oz = oracle_rows(x, gs, dtype)
    assert torch.equal(lv, ol) and torch.equal(sc, os_) and torch.equal(ze, oz)
    if dtype != torch.float32:
        assert torch.equal(kv8_dequantize(lv, sc, ze).float(), oracle_dequant(ol, os_, oz, gs, dtype).reshape(x.shape))


def test_kv8_quantize_rows_degenerate_groups_equal_the_fixture():
    """The groups of quantize_degenerate.npz (constant, nearly constant and extreme groups of 64): the reference's 8-bit levels,
    scale and zero without the solver."""
    d = np.load(os.path.join(HERE, "golden", "quantize_degenerate.npz"))
    x = torch.from_numpy(d["W"]).reshape(-1, 64)
    x = torch.cat([x, x], dim=1)  # rows of 128: two groups of 64 each
    lv, sc, ze = kv8_quantize_rows(x, 64)
    assert torch.equal(lv.reshape(-1, 64)[0::2], torch.from_numpy(d["b8_opt0/W_q"]))
    assert torch.equal(sc.reshape(-1, 1)[0::2], torch.from_numpy(d["b8_opt0/scale"]))
    assert torch.equal(ze.reshape(-1, 1)[0::2], torch.from_numpy(d["b8_opt0/zero"]))


def test_emulated_kv8_argument_checks(emu):
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = torch.zeros(1, dtype=torch.int64)

    def dec(hq, hkv, L, hd, gs, null=False):
        ptrs = [P(buf)] * 14
        ptrs[11] = P(p)
        if null:
            ptrs[6] = None
        return emu.hqq_b200_glue_rope_attn_decode_split_kv8(*ptrs, hq, hkv, L, hd, gs, 1, F16, None)

    def rows(hq, hkv, L, hd, gs, null=False):
        ptrs = [P(buf)] * 14
        if null:
            ptrs[12] = None
        return emu.hqq_b200_glue_rope_append_rows_kv8(*ptrs, 0, 1, hq, hkv, L, hd, gs, 1, F16, None)

    for fn, name in ((dec, b"hqq_b200_glue_rope_attn_decode_split_kv8"), (rows, b"hqq_b200_glue_rope_append_rows_kv8")):
        for hq, hkv, L, hd, gs in ((8, 1, 64, 64, 64), (8, 1, 64, 256, 64), (8, 1, 64, 128, 32), (8, 1, 64, 128, 256), (9, 1, 64, 128, 64),
                                   (16, 1, 64, 128, 64), (8, 1, 131073, 128, 64)):
            assert fn(hq, hkv, L, hd, gs) == E_UNSUPPORTED, (name, hq, hkv, L, hd, gs)
            assert name in emu.hqq_b200_last_error()
        assert fn(8, 1, 64, 128, 64, null=True) == E_INVALID
        assert name in emu.hqq_b200_last_error()
