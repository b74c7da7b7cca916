"""The 4-bit HQQ KV cache on the CPU kernel emulator (csrc/decode_glue.cu): the split-KV decode kernel and its _seqpos / _paged twins,
the five rows kernels, the two staging refills, the verify attention, the argument checks, and the framework-op format functions of
the decode harness against the CPU oracle.

The emulator has 4 SMs, so S = max(1, min(4 / n_kv, ceil(cache_len / 16))).  The decode output is held to the per-element bound of
tests/attn_split_ref.py against float64 attention over the dequantised cache (tests/attn_kv4_ref.py); cache rows to HQQ's
Quantizer.quantize(row, nbits=4, axis=1, optimize=False) packed by 4bit_u8, as the CPU oracle computes them, bit for bit.  The verify
attention writes each dequantised chunk into the tile the 16-bit form reads, so it must equal the 16-bit verify over the
dequantised cache bit for bit (that form is held to its bound in tests/test_spec_cpu.py)."""
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
import attn_kv4_ref as K4  # noqa: E402
import attn_split_ref as R  # noqa: E402
from hqq_b200.harness import KV_PAGE, kv8_dequantize, kv8_quantize_rows  # noqa: E402
from oracle import hqq_oracle as O  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
ONAME = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
SMS = 4
E_INVALID, E_UNSUPPORTED = -1, -2
VP, I = ctypes.c_void_p, ctypes.c_int
NAMES = ("kq", "ks", "kz", "vq", "vs", "vz")
LB = R.HD // 2  # packed level bytes a row


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    sig = {"hqq_b200_glue_rope_attn_decode_split_kv4": [VP] * 14 + [I] * 7, "hqq_b200_glue_rope_attn_decode_split_kv4_seqpos": [VP] * 14 + [I] * 7,
           "hqq_b200_glue_rope_attn_decode_split_kv4_paged": [VP] * 15 + [I] * 8, "hqq_b200_glue_rope_append_rows_kv4": [VP] * 14 + [I] * 9,
           "hqq_b200_glue_rope_append_rows_kv4_varlen": [VP] * 16 + [I] * 7, "hqq_b200_glue_rope_append_rows_kv4_paged": [VP] * 17 + [I] * 8,
           "hqq_b200_glue_kv4_stage": [VP] * 10 + [I] * 6, "hqq_b200_glue_kv4_stage_paged": [VP] * 11 + [I] * 7,
           "hqq_b200_glue_rope_append_rows_kv4_devpos": [VP] * 13 + [I] * 8, "hqq_b200_glue_rope_append_rows_kv4_devpos_paged": [VP] * 14 + [I] * 9,
           "hqq_b200_glue_attn_verify_split_kv4": [VP] * 10 + [I] * 8, "hqq_b200_glue_attn_verify_split_kv4_paged": [VP] * 11 + [I] * 9,
           "hqq_b200_glue_attn_verify_split": [VP] * 6 + [I] * 7, "hqq_b200_glue_rope_append_rows": [VP] * 8 + [I] * 8}
    for n, a in sig.items():
        getattr(lib, n).argtypes = a + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def ints(xs):
    return (ctypes.c_int * len(xs))(*xs)


def oracle_rows(x, gs, dtype):
    """oracle.quantize(nbits=4, optimize=False) of each row (float32 of the T values), packed by the oracle's 4bit_u8: levels uint8
    [..., 64], scale and zero cast to T."""
    rows = x.reshape(-1, R.HD).float().numpy()
    lv, sc, ze = [], [], []
    for r in rows:
        W_q, meta = O.quantize(r.reshape(1, -1), nbits=4, group_size=gs, axis=1, optimize=False, bitpack=True)
        lv.append(np.asarray(W_q).reshape(-1).astype(np.uint8))
        sc.append(np.asarray(meta["scale"]).reshape(-1))
        ze.append(np.asarray(meta["zero"]).reshape(-1))
    shape = x.shape[:-1]
    ng = R.HD // gs
    return (torch.from_numpy(np.stack(lv)).reshape(shape + (LB,)), torch.from_numpy(np.stack(sc)).to(dtype).reshape(shape + (ng,)),
            torch.from_numpy(np.stack(ze)).to(dtype).reshape(shape + (ng,)))


def oracle_dequant(lv, scale, zero, gs, dtype):
    """oracle.dequantize of packed 4-bit rows with the meta in T: float32 values of T, [rows, 128]."""
    out = []
    for w, s, z in zip(lv.reshape(-1, LB).numpy(), scale.reshape(-1, R.HD // gs).float().numpy(), zero.reshape(-1, R.HD // gs).float().numpy()):
        meta = {"packing": "4bit_u8", "nbits": 4, "group_size": gs, "axis": 1, "shape": (1, R.HD), "scale": s.reshape(-1, 1), "zero": z.reshape(-1, 1)}
        out.append(np.asarray(O.dequantize(w.reshape(-1, gs), meta, ONAME[dtype]), dtype=np.float32).reshape(-1))
    return torch.from_numpy(np.stack(out)) if out else torch.zeros(0, R.HD)


def random_caches(gen, lead, gs, dtype):
    """Random 4-bit caches [*lead, 64] levels and [*lead, 128 / gs] meta in the range kv8_quantize_rows(bits=4) produces."""
    ng = R.HD // gs
    c = {n: torch.randint(0, 256, lead + (LB,), generator=gen, dtype=torch.uint8) for n in ("kq", "vq")}
    for n in ("ks", "vs"):
        c[n] = (torch.rand(lead + (ng,), generator=gen) * 0.3 + 0.05).to(dtype)
    for n in ("kz", "vz"):
        c[n] = (torch.rand(lead + (ng,), generator=gen) * 15).to(dtype)
    return c


def scrambled(gen, B, L):
    """A table [B, L / 64] over exactly B L / 64 pages in a random physical order."""
    E = L // KV_PAGE
    return torch.randperm(B * E, generator=gen).view(B, E).to(torch.int32).contiguous(), B * E


def to_pool(cache, tab, N):
    """The pool [N + 1, hkv, 64, X] holding the contiguous cache [B, hkv, L, X] through tab; the sink 0xFF / NaN."""
    B, hkv, L, X = cache.shape
    pool = torch.full((N + 1, hkv, KV_PAGE, X), 255 if cache.dtype == torch.uint8 else float("nan"), dtype=cache.dtype)
    for b in range(B):
        for j in range(L // KV_PAGE):
            pool[int(tab[b, j])] = cache[b, :, j * KV_PAGE:(j + 1) * KV_PAGE]
    return pool


def gather(pool, tab):
    B, E = tab.shape
    return pool[tab.long()].permute(0, 2, 1, 3, 4).reshape(B, pool.shape[1], E * KV_PAGE, pool.shape[3]).contiguous()


def run_decode(emu, case, pos, cos, sin, hq, hkv, dtype, gs, kind="fixed", tab=None, N=0):
    """One decode launch: pos an int (fixed) or a list (seqpos / paged, case caches then being pools for paged)."""
    batch = case["q"].shape[0]
    L = cos.shape[0]
    c = {n: case[n].clone() for n in NAMES}
    out = torch.zeros(batch, hq * R.HD, dtype=dtype)
    ws = torch.zeros(R.workspace_bytes(SMS, hq, hkv, batch), dtype=torch.uint8)
    p = torch.tensor(pos if isinstance(pos, list) else [pos], dtype=torch.int64)
    args = [P(case["q"]), P(case["k"]), P(case["v"]), P(cos), P(sin)] + [P(c[n]) for n in NAMES]
    tail = [P(p), P(out), P(ws), hq, hkv, L, R.HD, gs, batch]
    if kind == "fixed":
        rc = emu.hqq_b200_glue_rope_attn_decode_split_kv4(*args, *tail, CODE[dtype], None)
    elif kind == "seqpos":
        rc = emu.hqq_b200_glue_rope_attn_decode_split_kv4_seqpos(*args, *tail, CODE[dtype], None)
    else:
        rc = emu.hqq_b200_glue_rope_attn_decode_split_kv4_paged(*args, P(tab), *tail, N, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, c, ws


def positions(L, S):
    c = R.TILE * max(1, (L // (2 * S)) // R.TILE)  # a chunk length whose S-fold fits the cache twice
    return sorted({0, 15, 16, 17, S * c - 1, S * c, S * c + 1, L - 1})


CASES = [(hq, hkv, B) for (hq, hkv) in ((2, 2), (8, 2), (8, 1)) for B in (1, 3)]


@pytest.mark.parametrize("gs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv,B", CASES)
def test_emulated_kv4_attention_within_bound_and_row_pos_exact(emu, dtype, gs, hq, hkv, B):
    """Output within the bound over the dequantised cache (row pos = dequant(quant(rope(k)))) at tile and chunk edges; the row
    written at pos equals the oracle bit for bit and no other byte changes; tickets back at zero; the five defects break the bound."""
    L = 300
    S = R.split_count(SMS, hkv, L)
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(1000 * hq + 100 * hkv + 10 * B + gs)
    for pos in positions(L, S):
        case = K4.make_case(gen, B, hq, hkv, L, pos, dtype, cos, sin, gs, "cpu")
        out, c, ws = run_decode(emu, case, pos, cos, sin, hq, hkv, dtype, gs)
        y, bound, exp = K4.reference(case, pos, cos, sin, S, dtype, gs)
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
            for name, bad in K4.defects(case, exp, pos, cos, sin, S, gs).items():
                if name == "neighbouring group's scale" and gs != 32:
                    continue
                assert not R.within(bad, y, bound)[1], (pos, name)


@pytest.mark.parametrize("gs,dtype", [(32, torch.float16), (64, torch.bfloat16)], ids=["gs32-f16", "gs64-bf16"])
def test_emulated_kv4_seqpos_and_paged_equal_fixed(emu, gs, dtype):
    """_seqpos at equal positions equals the fixed kernel bit for bit; at different positions each sequence equals the fixed kernel
    run on it alone; _paged over a scrambled table equals _seqpos on the gathered cache (output, pools, tickets)."""
    hq, hkv, B, L = 8, 2, 3, 192
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(gs)
    case = K4.make_case(gen, B, hq, hkv, L, 100, dtype, cos, sin, gs, "cpu")
    fixed = run_decode(emu, case, 100, cos, sin, hq, hkv, dtype, gs)
    seq = run_decode(emu, case, [100] * B, cos, sin, hq, hkv, dtype, gs, "seqpos")
    assert torch.equal(fixed[0], seq[0]) and all(torch.equal(fixed[1][n], seq[1][n]) for n in NAMES)
    pos = [0, 64, L - 1]
    seq = run_decode(emu, case, pos, cos, sin, hq, hkv, dtype, gs, "seqpos")
    for b, p in enumerate(pos):
        one = {n: case[n][b:b + 1] for n in case if n not in ("kc", "vc")}
        o1, c1, _ = run_decode(emu, one, p, cos, sin, hq, hkv, dtype, gs)
        assert torch.equal(seq[0][b:b + 1], o1) and all(torch.equal(seq[1][n][b:b + 1], c1[n]) for n in NAMES), b
    tab, N = scrambled(gen, B, L)
    pooled = dict(case)
    for n in NAMES:
        pooled[n] = to_pool(case[n], tab, N)
    out, c, ws = run_decode(emu, pooled, pos, cos, sin, hq, hkv, dtype, gs, "paged", tab, N)
    assert torch.equal(out, seq[0]) and torch.count_nonzero(ws[-4 * B * hkv:]) == 0
    for n in NAMES:
        assert torch.equal(gather(c[n], tab), seq[1][n]), n
        assert torch.equal(c[n][N].view(torch.uint8), pooled[n][N].view(torch.uint8)), n  # the sink untouched


def rows_data(gen, B, T, hq, hkv, dtype):
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    return rn(B * T, hq * R.HD), rn(B * T, hkv * R.HD), rn(B * T, hkv * R.HD)


@pytest.mark.parametrize("gs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_kv4_rows_kernel_matches_decode_rows_oracle_and_q(emu, dtype, gs):
    """The rows kernel writes the cache rows the decode kernel writes from the same k and v (and the oracle's), stages
    oracle.dequantize of them, leaves every other row alone, and its q_out equals hqq_b200_glue_rope_append_rows' bit for bit."""
    hq, hkv, B, L, T, pos0 = 8, 2, 3, 96, 20, 33
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(gs + CODE[dtype])
    q, k, v = rows_data(gen, B, T, hq, hkv, dtype)
    c0 = random_caches(gen, (B, hkv, L), gs, dtype)
    kst, vst = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype), torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
    c = {n: t.clone() for n, t in c0.items()}
    st = [kst.clone(), vst.clone()]
    qo = torch.zeros(B * T, hq * R.HD, dtype=dtype)
    rc = emu.hqq_b200_glue_rope_append_rows_kv4(P(q), P(k), P(v), P(cos), P(sin), *[P(c[n]) for n in NAMES], P(st[0]), P(st[1]), P(qo), pos0, T, hq,
                                                hkv, L, R.HD, gs, B, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    qx, kx, vx = torch.zeros_like(qo), torch.zeros(B, hkv, L, R.HD, dtype=dtype), torch.zeros(B, hkv, L, R.HD, dtype=dtype)
    assert emu.hqq_b200_glue_rope_append_rows(P(q), P(k), P(v), P(cos), P(sin), P(kx), P(vx), P(qx), pos0, T, hq, hkv, L, R.HD, B, CODE[dtype], None) == 0
    assert torch.equal(qo, qx)
    rows = slice(pos0, pos0 + T)
    outside = torch.ones(L, dtype=torch.bool)
    outside[rows] = False
    for side, stg, stg0, x in (("k", st[0], kst, kx), ("v", st[1], vst, vx)):
        ol, os_, oz = oracle_rows(x[:, :, rows], gs, dtype)
        assert torch.equal(c[side + "q"][:, :, rows], ol) and torch.equal(c[side + "s"][:, :, rows], os_) and torch.equal(c[side + "z"][:, :, rows], oz)
        for n in ("q", "s", "z"):
            assert torch.equal(c[side + n][:, :, outside], c0[side + n][:, :, outside])
        assert torch.equal(stg[:, :, outside], stg0[:, :, outside])
        assert torch.equal(stg[:, :, rows].float().reshape(-1, R.HD), oracle_dequant(ol, os_, oz, gs, dtype))
    for t in (0, T - 1):  # the decode kernel's row at each end of the chunk from the same k and v
        p = pos0 + t
        case = {"q": q.view(B, T, -1)[:, t].contiguous(), "k": k.view(B, T, -1)[:, t].contiguous(), "v": v.view(B, T, -1)[:, t].contiguous(), **c0}
        _, d, _ = run_decode(emu, case, p, cos, sin, hq, hkv, dtype, gs)
        for n in NAMES:
            assert torch.equal(d[n][:, :, p], c[n][:, :, p]), (t, n)


@pytest.mark.parametrize("gs,dtype", [(32, torch.bfloat16), (64, torch.float16)], ids=["gs32-bf16", "gs64-f16"])
def test_emulated_kv4_rows_twins_and_staging(emu, gs, dtype):
    """_varlen equals the fixed kernel slot by slot; _paged equals _varlen on the gathered cache; _devpos equals _varlen's cache rows
    and q_out (rows past the cache end skipped); _devpos_paged equals _devpos on the gathered cache; both staging refills equal
    oracle.dequantize of the cache rows [0, pos0) and touch nothing else."""
    hq, hkv, B, L = 8, 2, 3, 192
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(7 + gs)
    pos0, n_tok = [5, 0, 130], [40, 0, 62]
    rows = sum(n_tok)
    q, k, v = rows_data(gen, 1, rows, hq, hkv, dtype)
    c0 = random_caches(gen, (B, hkv, L), gs, dtype)
    stage0 = [torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype) for _ in range(2)]

    def varlen(c, st, qo):
        assert emu.hqq_b200_glue_rope_append_rows_kv4_varlen(P(q), P(k), P(v), P(cos), P(sin), *[P(c[n]) for n in NAMES], P(st[0]), P(st[1]), P(qo),
                                                             ints(pos0), ints(n_tok), hq, hkv, L, R.HD, gs, B, CODE[dtype], None) == 0, emu.hqq_b200_last_error()

    cv, sv, qv = {n: t.clone() for n, t in c0.items()}, [t.clone() for t in stage0], torch.zeros(rows, hq * R.HD, dtype=dtype)
    varlen(cv, sv, qv)
    r0 = 0
    for b in range(B):  # slot by slot against the fixed-length kernel on that slot alone
        if n_tok[b]:
            cf = {n: c0[n][b:b + 1].clone() for n in NAMES}
            sf = [t[b:b + 1].clone() for t in stage0]
            qf = torch.zeros(n_tok[b], hq * R.HD, dtype=dtype)
            sl = slice(r0, r0 + n_tok[b])
            assert emu.hqq_b200_glue_rope_append_rows_kv4(P(q[sl].contiguous()), P(k[sl].contiguous()), P(v[sl].contiguous()), P(cos), P(sin),
                                                          *[P(cf[n]) for n in NAMES], P(sf[0]), P(sf[1]), P(qf), pos0[b], n_tok[b], hq, hkv, L, R.HD,
                                                          gs, 1, CODE[dtype], None) == 0
            assert torch.equal(qf, qv[sl]) and all(torch.equal(cf[n][0], cv[n][b]) for n in NAMES)
            assert all(torch.equal(sf[i][0], sv[i][b]) for i in range(2))
            r0 += n_tok[b]
        else:
            assert all(torch.equal(cv[n][b], c0[n][b]) for n in NAMES)
    # paged against varlen, on a scrambled table
    tab, N = scrambled(gen, B, L)
    pools = {n: to_pool(c0[n], tab, N) for n in NAMES}
    sp, qp = [t.clone() for t in stage0], torch.zeros_like(qv)
    assert emu.hqq_b200_glue_rope_append_rows_kv4_paged(P(q), P(k), P(v), P(cos), P(sin), *[P(pools[n]) for n in NAMES], P(tab), P(sp[0]), P(sp[1]),
                                                        P(qp), ints(pos0), ints(n_tok), hq, hkv, L, R.HD, gs, B, N, CODE[dtype], None) == 0
    assert torch.equal(qp, qv) and all(torch.equal(sp[i], sv[i]) for i in range(2))
    assert all(torch.equal(gather(pools[n], tab), cv[n]) for n in NAMES)
    # the staging refills: rows [0, pos0) of the slots in the chunk, oracle.dequantize of the cache rows
    for paged in (False, True):
        st = [t.clone() for t in stage0]
        if paged:
            rc = emu.hqq_b200_glue_kv4_stage_paged(*[P(pools[n]) for n in NAMES], P(tab), P(st[0]), P(st[1]), ints(pos0), ints(n_tok), hkv, L, R.HD, gs,
                                                   B, N, CODE[dtype], None)
        else:
            rc = emu.hqq_b200_glue_kv4_stage(*[P(cv[n]) for n in NAMES], P(st[0]), P(st[1]), ints(pos0), ints(n_tok), hkv, L, R.HD, gs, B, CODE[dtype],
                                             None)
        assert rc == 0, emu.hqq_b200_last_error()
        for b in range(B):
            p = pos0[b] if n_tok[b] else 0
            for i, side in enumerate("kv"):
                want = oracle_dequant(cv[side + "q"][b, :, :p], cv[side + "s"][b, :, :p], cv[side + "z"][b, :, :p], gs, dtype)
                assert torch.equal(st[i][b, :, :p].float().reshape(-1, R.HD), want), (paged, b, side)
                assert torch.equal(st[i][b, :, p:], stage0[i][b, :, p:]), (paged, b, side)
    # the device-position appends: T rows per slot at pos[b], the ones past the cache end skipped
    T, dpos = 4, [3, 70, L - 2]
    qd, kd, vd = rows_data(gen, B, T, hq, hkv, dtype)
    cd, qod = {n: t.clone() for n, t in c0.items()}, torch.zeros(B * T, hq * R.HD, dtype=dtype)
    p64 = torch.tensor(dpos, dtype=torch.int64)
    assert emu.hqq_b200_glue_rope_append_rows_kv4_devpos(P(qd), P(kd), P(vd), P(cos), P(sin), *[P(cd[n]) for n in NAMES], P(qod), P(p64), T, hq, hkv,
                                                         L, R.HD, gs, B, CODE[dtype], None) == 0, emu.hqq_b200_last_error()
    fit = [min(T, L - p) for p in dpos]
    keep = torch.cat([torch.arange(b * T, b * T + fit[b]) for b in range(B)])
    cx, sx, qx = {n: t.clone() for n, t in c0.items()}, [t.clone() for t in stage0], torch.zeros(len(keep), hq * R.HD, dtype=dtype)
    assert emu.hqq_b200_glue_rope_append_rows_kv4_varlen(P(qd[keep].contiguous()), P(kd[keep].contiguous()), P(vd[keep].contiguous()), P(cos), P(sin),
                                                         *[P(cx[n]) for n in NAMES], P(sx[0]), P(sx[1]), P(qx), ints(dpos), ints(fit), hq, hkv, L, R.HD,
                                                         gs, B, CODE[dtype], None) == 0
    assert torch.equal(qod[keep], qx) and all(torch.equal(cd[n], cx[n]) for n in NAMES)
    pd = {n: to_pool(c0[n], tab, N) for n in NAMES}
    qpd = torch.zeros_like(qod)
    assert emu.hqq_b200_glue_rope_append_rows_kv4_devpos_paged(P(qd), P(kd), P(vd), P(cos), P(sin), *[P(pd[n]) for n in NAMES], P(tab), P(qpd), P(p64),
                                                               T, hq, hkv, L, R.HD, gs, B, N, CODE[dtype], None) == 0
    assert torch.equal(qpd, qod) and all(torch.equal(gather(pd[n], tab), cd[n]) for n in NAMES)


def verify_ws(hq, hkv, T, B):
    g = B * hkv * -(-T * (hq // hkv) // 16)
    return g * max(1, SMS // hkv) * 16 * 130 * 4 + g * 4


@pytest.mark.parametrize("dtype,heads,T,gs", [(torch.float16, (8, 2), 4, 32), (torch.bfloat16, (8, 1), 8, 64), (torch.bfloat16, (2, 2), 2, 32)],
                         ids=["f16-G4-T4-gs32", "bf16-G8-T8-gs64", "bf16-G1-T2-gs32"])
def test_emulated_verify_attention_kv4_equals_16bit_form_and_paged_equal(emu, dtype, heads, T, gs):
    """The 4-bit verify equals the 16-bit verify over the dequantised cache bit for bit (the same tile, MMAs and merge after the
    dequantisation), tickets back at zero, and the paged twin equal bit for bit."""
    hq, hkv = heads
    B, L = 2, 192
    gen = torch.Generator().manual_seed(T + gs)
    c = random_caches(gen, (B, hkv, L), gs, dtype)
    q = torch.randn(B * T, hq * R.HD, generator=gen).to(dtype)
    pos = [0, L - T - 3]
    p64 = torch.tensor(pos, dtype=torch.int64)
    kd, vd = (kv8_dequantize(c[s + "q"], c[s + "s"], c[s + "z"], 4).contiguous() for s in "kv")
    want = torch.zeros(B * T, hq * R.HD, dtype=dtype)
    ws = torch.zeros(verify_ws(hq, hkv, T, B), dtype=torch.uint8)
    assert emu.hqq_b200_glue_attn_verify_split(P(q), P(kd), P(vd), P(p64), P(want), P(ws), hq, hkv, L, R.HD, T, B, CODE[dtype], None) == 0
    got = torch.zeros_like(want)
    ws = torch.zeros_like(ws)
    assert emu.hqq_b200_glue_attn_verify_split_kv4(P(q), *[P(c[n]) for n in NAMES], P(p64), P(got), P(ws), hq, hkv, L, R.HD, gs, T, B, CODE[dtype],
                                                   None) == 0, emu.hqq_b200_last_error()
    assert torch.equal(got, want)
    assert torch.count_nonzero(ws[-4 * B * hkv * -(-T * (hq // hkv) // 16):]) == 0
    tab, N = scrambled(gen, B, L)
    pools = {n: to_pool(c[n], tab, N) for n in NAMES}
    gp = torch.zeros_like(want)
    assert emu.hqq_b200_glue_attn_verify_split_kv4_paged(P(q), *[P(pools[n]) for n in NAMES], P(tab), P(p64), P(gp), P(torch.zeros_like(ws)), hq, hkv,
                                                         L, R.HD, gs, T, B, N, CODE[dtype], None) == 0
    assert torch.equal(gp, want)


@pytest.mark.parametrize("gs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
def test_kv4_quantize_rows_equals_oracle(dtype, gs):
    """kv8_quantize_rows(bits=4) on random rows, rows of large and small magnitude, a constant group and a group whose range is below
    1e-4 equals oracle.quantize(..., nbits=4, axis=1, optimize=False) packed by 4bit_u8, meta cast to T; kv8_dequantize(bits=4)
    equals oracle.dequantize; and the 8-bit default is unchanged."""
    gen = torch.Generator().manual_seed(gs)
    x = torch.cat([torch.randn(64, R.HD, generator=gen), torch.randn(16, R.HD, generator=gen).clamp(-6, 6) * 1e4, torch.randn(16, R.HD, generator=gen) * 1e-3])
    x[0, :gs] = 0.75                                          # a constant group
    x[1, gs:2 * gs] = 1.0 + torch.arange(gs) * 1e-6           # a range below 1e-4
    x = x.to(dtype)
    lv, sc, ze = kv8_quantize_rows(x, gs, 4)
    ol, os_, oz = oracle_rows(x, gs, dtype)
    assert lv.shape == (x.shape[0], LB)
    assert torch.equal(lv, ol) and torch.equal(sc, os_) and torch.equal(ze, oz)
    if dtype != torch.float32:
        assert torch.equal(kv8_dequantize(lv, sc, ze, 4).float(), oracle_dequant(ol, os_, oz, gs, dtype))


def test_kv4_packing_is_the_reference_4bit_u8_layout():
    """Byte d of a packed row holds level d in its high nibble and level d + 64 in its low nibble, as BitPack.pack_4bit_u8 of the
    row's [128 / gs, gs] levels gives it for gs 32 and 64."""
    for gs in (32, 64):
        q = torch.randint(0, 16, (5, R.HD), generator=torch.Generator().manual_seed(gs), dtype=torch.uint8)
        ref = np.stack([np.asarray(O.pack_4bit_u8(r.numpy().reshape(-1, gs))).reshape(-1) for r in q])
        assert torch.equal(torch.from_numpy(ref), (q[:, :64] << 4) | q[:, 64:])


def test_emulated_kv4_argument_checks(emu):
    """Every 4-bit entry point rejects what its kv8 twin rejects, and group sizes outside {32, 64}."""
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = torch.zeros(1, dtype=torch.int64)
    tab = torch.zeros(2, dtype=torch.int32)
    one, zero = ints([1]), ints([0])
    b = P(buf)

    def dec(hq, hkv, L, hd, gs, null=False):
        ptrs = [b] * 14
        ptrs[11] = P(p)
        if null:
            ptrs[6] = None
        return emu.hqq_b200_glue_rope_attn_decode_split_kv4(*ptrs, hq, hkv, L, hd, gs, 1, F16, None)

    def rows(hq, hkv, L, hd, gs, null=False):
        ptrs = [b] * 14
        if null:
            ptrs[12] = None
        return emu.hqq_b200_glue_rope_append_rows_kv4(*ptrs, 0, 1, hq, hkv, L, hd, gs, 1, F16, None)

    def stage(hq, hkv, L, hd, gs, null=False):
        ptrs = [b] * 8
        if null:
            ptrs[6] = None
        return emu.hqq_b200_glue_kv4_stage(*ptrs, one, one, hkv, L, hd, gs, 1, F16, None)

    def verify(hq, hkv, L, hd, gs, null=False):
        ptrs = [b] * 10
        ptrs[7] = P(p)
        if null:
            ptrs[2] = None
        return emu.hqq_b200_glue_attn_verify_split_kv4(*ptrs, hq, hkv, L, hd, gs, 1, 1, F16, None)

    for fn, name in ((dec, b"hqq_b200_glue_rope_attn_decode_split_kv4"), (rows, b"hqq_b200_glue_rope_append_rows_kv4"), (stage, b"hqq_b200_glue_kv4_stage"),
                     (verify, b"hqq_b200_glue_attn_verify_split_kv4")):
        for gs in (16, 128, 256):
            assert fn(8, 1, 64, 128, gs) == E_UNSUPPORTED, (name, gs)
            assert name in emu.hqq_b200_last_error()
        if fn is not stage:
            for hq, hkv, L, hd in ((8, 1, 64, 64), (8, 1, 64, 256), (9, 1, 64, 128)):
                assert fn(hq, hkv, L, hd, 64) != 0, (name, hq, hkv, L, hd)
        assert fn(8, 1, 64, 128, 64, null=True) == E_INVALID
        assert name in emu.hqq_b200_last_error()
    # the paged forms: a null table, cache_len not a multiple of 64, n_pages < 1
    for bad in ((None, 64, 1), (P(tab), 96, 1), (P(tab), 64, 0)):
        t, L, n = bad
        assert emu.hqq_b200_glue_rope_attn_decode_split_kv4_paged(*[b] * 11, t, P(p), b, b, 8, 1, L, 128, 64, 1, n, F16, None) == E_INVALID
        assert emu.hqq_b200_glue_rope_append_rows_kv4_paged(*[b] * 11, t, b, b, b, one, one, 8, 1, L, 128, 64, 1, n, F16, None) == E_INVALID
        assert emu.hqq_b200_glue_kv4_stage_paged(*[b] * 6, t, b, b, one, zero, 2, L, 128, 64, 1, n, F16, None) == E_INVALID
        assert emu.hqq_b200_glue_rope_append_rows_kv4_devpos_paged(*[b] * 11, t, b, P(p), 1, 8, 1, L, 128, 64, 1, n, F16, None) == E_INVALID
        assert emu.hqq_b200_glue_attn_verify_split_kv4_paged(*[b] * 7, t, P(p), b, b, 8, 1, L, 128, 64, 1, 1, n, F16, None) == E_INVALID


def test_kv4_model_options_rejected_before_any_allocation():
    """DecodeModel(kv_bits=4) needs an explicit kv_group_size of 32 or 64; kv_bits outside {16, 8, 4} and the 8-bit group sizes keep
    their checks.  All of them raise ValueError before the model touches a device."""
    from hqq_b200 import harness
    shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=1, n_heads=8, n_kv_heads=2, vocab=2048)
    for kw in ({"kv_bits": 4}, {"kv_bits": 4, "kv_group_size": 128}, {"kv_bits": 4, "kv_group_size": 16}, {"kv_bits": 2},
               {"kv_bits": 8, "kv_group_size": 32}, {"kv_group_size": 256}):
        with pytest.raises(ValueError):
            harness.DecodeModel(shape, dtype=torch.float16, device="cpu", cache_len=64, **kw)
