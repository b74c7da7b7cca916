"""Paged KV cache on the CPU kernel emulator and the page allocator (csrc/decode_glue.cu PAGED instantiations, harness.PageAllocator).

Every _paged entry point is held bit for bit to its contiguous ragged counterpart (_seqpos / _varlen) run on the cache gathered
through the page table: output, every cache row and the tickets.  The tables are scrambled -- physical order differs from logical
order, some full pages are shared by two slots for reading, entries past a slot's rows point at the sink -- and the pools start
as random bytes, the sink as NaN, so every page holds different data: swapping two table entries changes the output, and a row
read from the wrong page cannot go unnoticed.  Every byte of the pools outside the rows a call writes must come out unchanged."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import attn_split_ref as R  # noqa: E402
from hqq_b200.harness import KV_PAGE, PageAllocator  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
SMS = 4
E_INVALID = -1
VP, I = ctypes.c_void_p, ctypes.c_int
G1, G4, G8 = (2, 2), (8, 2), (8, 1)  # (n_q, n_kv) heads for G = 1, 4, 8
F, BF = torch.float16, torch.bfloat16
DT_ID = {F: "f16", BF: "bf16"}
PG = KV_PAGE
# The emulator's cost grows with the CTAs it runs, so the cases cover every kernel in both dtypes and, across them, every G and group
# size, rather than the full cross product.


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    sig = {"hqq_b200_glue_rope_attn_decode_batch_seqpos": [VP] * 9 + [I] * 6, "hqq_b200_glue_rope_attn_decode_split_seqpos": [VP] * 10 + [I] * 6,
           "hqq_b200_glue_rope_attn_decode_split_kv8_seqpos": [VP] * 14 + [I] * 7, "hqq_b200_glue_rope_append_rows_varlen": [VP] * 10 + [I] * 6,
           "hqq_b200_glue_rope_append_rows_kv8_varlen": [VP] * 16 + [I] * 7, "hqq_b200_glue_attn_prefill_varlen": [VP] * 6 + [I] * 6,
           "hqq_b200_glue_rope_attn_decode_batch_paged": [VP] * 10 + [I] * 7, "hqq_b200_glue_rope_attn_decode_split_paged": [VP] * 11 + [I] * 7,
           "hqq_b200_glue_rope_attn_decode_split_kv8_paged": [VP] * 15 + [I] * 8, "hqq_b200_glue_rope_append_rows_paged": [VP] * 11 + [I] * 7,
           "hqq_b200_glue_rope_append_rows_kv8_paged": [VP] * 17 + [I] * 8, "hqq_b200_glue_kv8_stage_paged": [VP] * 11 + [I] * 7,
           "hqq_b200_glue_attn_prefill_paged": [VP] * 7 + [I] * 7}
    for n, a in sig.items():
        getattr(lib, n).argtypes = a + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def ints(xs):
    return (ctypes.c_int * len(xs))(*xs)


# ------------------------------------------------------------------------------------------------------------------ tables and pools
def scrambled_table(gen, ends, entries, shared=True):
    """A table [B, entries] int32 over a pool of N + 1 pages: slot b owns pages for entries 0 .. (ends[b] - 1) / 64 in a random
    physical order; with `shared`, the first full page of each slot after the first is replaced by the previous slot's (both read
    it); entries past the last one point at the sink N.  ends[b] = the first position slot b does not hold (its pos + 1)."""
    B = len(ends)
    need = [-(-e // PG) for e in ends]
    N = sum(need) + 3  # a few pages no slot holds
    perm = torch.randperm(N, generator=gen).tolist()
    tab = torch.full((B, entries), N, dtype=torch.int32)
    k = 0
    for b in range(B):
        for j in range(need[b]):
            tab[b, j] = perm[k]
            k += 1
    if shared:
        for b in range(1, B):
            # full pages below the rows slot b writes: entries j with 64 (j + 1) <= its first written row (ends[b] - 1 for decode)
            if (ends[b] - 1) // PG >= 1 and (ends[b - 1] - 1) // PG >= 1:
                tab[b, 0] = tab[b - 1, 0]
    return tab, N


def pools(gen, N, hkv, dtype, gs=None):
    """Random pools [N + 1, hkv, 64, 128] (kv8: uint8 levels and meta [.., 128 / gs]); the sink page NaN (levels 0xFF)."""
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    if gs is None:
        p = {"kc": rn(N + 1, hkv, PG, R.HD), "vc": rn(N + 1, hkv, PG, R.HD)}
        for t in p.values():
            t[N] = float("nan")
        return p
    ng = R.HD // gs
    p = {"kq": torch.randint(0, 256, (N + 1, hkv, PG, R.HD), generator=gen, dtype=torch.uint8),
         "vq": torch.randint(0, 256, (N + 1, hkv, PG, R.HD), generator=gen, dtype=torch.uint8)}
    for n in ("ks", "vs"):
        p[n] = (torch.rand(N + 1, hkv, PG, ng, generator=gen) * 0.02 + 0.005).to(dtype)
    for n in ("kz", "vz"):
        p[n] = (torch.rand(N + 1, hkv, PG, ng, generator=gen) * 255).to(dtype)
    for n, t in p.items():
        t[N] = 255 if t.dtype == torch.uint8 else float("nan")
    return p


def gather(pool, tab):
    """The contiguous cache [B, hkv, L, X] the table describes."""
    B, E = tab.shape
    return pool[tab.long()].permute(0, 2, 1, 3, 4).reshape(B, pool.shape[1], E * PG, pool.shape[3]).contiguous()


def written_mask(pool, tab, rows_of):
    """Bool mask [N + 1, hkv, 64] of the pool rows a call writes: rows_of[b] = the positions slot b writes."""
    m = torch.zeros(pool.shape[:3], dtype=torch.bool)
    for b, ps in enumerate(rows_of):
        for p in ps:
            m[int(tab[b, p // PG]), :, p % PG] = True
    return m


def check_pools(before, after, unpaged_after, tab, rows_of):
    """Pool rows the call writes equal the contiguous call's rows through the table; every other byte is unchanged."""
    for n in before:
        m = written_mask(before[n], tab, rows_of)
        a, b0 = after[n].view(torch.uint8) if after[n].dtype != torch.uint8 else after[n], before[n]
        b0 = b0.view(torch.uint8) if b0.dtype != torch.uint8 else b0
        assert torch.equal(a[~m], b0[~m]), n
        g = gather(after[n], tab)
        for b, ps in enumerate(rows_of):
            for p in ps:
                assert torch.equal(g[b, :, p].view(torch.uint8) if g.dtype != torch.uint8 else g[b, :, p],
                                   unpaged_after[n][b, :, p].view(torch.uint8) if g.dtype != torch.uint8 else unpaged_after[n][b, :, p]), (n, b, p)


# ------------------------------------------------------------------------------------------------------------------ decode
L_DEC = 192
POS = [0, 63, 64, 65, 127, 128, L_DEC - 1]
DEC_NAMES = {"batch": ("kc", "vc"), "split": ("kc", "vc"), "kv8": ("kq", "ks", "kz", "vq", "vs", "vz")}
DEC_FN = {"batch": "hqq_b200_glue_rope_attn_decode_batch", "split": "hqq_b200_glue_rope_attn_decode_split",
          "kv8": "hqq_b200_glue_rope_attn_decode_split_kv8"}


def run_decode(emu, kind, paged, qkv, caches, tab, N, pos, cos, sin, hq, hkv, dtype, gs):
    B = qkv["q"].shape[0]
    c = {n: t.clone() for n, t in caches.items()}
    out = torch.zeros(B, hq * R.HD, dtype=dtype)
    p = torch.tensor(pos, dtype=torch.int64)
    ws = torch.zeros(R.workspace_bytes(SMS, hq, hkv, B), dtype=torch.uint8)
    head = [P(qkv["q"]), P(qkv["k"]), P(qkv["v"]), P(cos), P(sin)] + [P(c[n]) for n in DEC_NAMES[kind]]
    fn = getattr(emu, DEC_FN[kind] + ("_paged" if paged else "_seqpos"))
    mid = ([P(tab)] if paged else []) + [P(p), P(out)] + ([] if kind == "batch" else [P(ws)])
    tail = [hq, hkv, L_DEC, R.HD] + ([gs] if kind == "kv8" else []) + [B] + ([N] if paged else []) + [CODE[dtype], None]
    rc = fn(*head, *mid, *tail)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, c, ws[-4 * B * hkv:]


DECODE_CASES = [("batch", None, F, G1), ("batch", None, BF, G8), ("split", None, F, G4), ("split", None, BF, G1), ("kv8", 64, F, G8),
                ("kv8", 64, BF, G4), ("kv8", 128, F, G1), ("kv8", 128, BF, G8)]


@pytest.mark.parametrize("kind,gs,dtype,heads", DECODE_CASES, ids=[f"{k}{gs or ''}-{DT_ID[d]}-G{h[0] // h[1]}" for k, gs, d, h in DECODE_CASES])
def test_emulated_paged_decode_equals_seqpos_on_gathered_cache(emu, kind, gs, dtype, heads):
    """Positions 0, 63, 64, 65, 127, 128 and cache_len - 1 in one launch over a scrambled table: output, tickets and written rows
    equal the _seqpos kernel on the gathered cache bit for bit; nothing else in the pools changes; swapping a slot's full and partial
    page changes its output."""
    hq, hkv = heads
    gen = torch.Generator().manual_seed(7 * hq + hkv + CODE[dtype] + (gs or 0) + len(kind))
    cos, sin = R.tables(L_DEC, dtype, "cpu")
    B = len(POS)
    tab, N = scrambled_table(gen, [p + 1 for p in POS], L_DEC // PG)
    pool = pools(gen, N, hkv, dtype, gs)
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    qkv = {"q": rn(B, hq * R.HD), "k": rn(B, hkv * R.HD), "v": rn(B, hkv * R.HD)}
    out, after, tk = run_decode(emu, kind, True, qkv, pool, tab, N, POS, cos, sin, hq, hkv, dtype, gs)
    flat = {n: gather(t, tab) for n, t in pool.items()}
    ref, ref_after, tk_ref = run_decode(emu, kind, False, qkv, flat, None, N, POS, cos, sin, hq, hkv, dtype, gs)
    assert torch.equal(out, ref)
    assert torch.count_nonzero(tk) == 0 and torch.count_nonzero(tk_ref) == 0
    check_pools(pool, after, ref_after, tab, [[p] for p in POS])
    b = POS.index(65)  # its full page 0 and partial page 1 trade places: the attended rows change (attention is blind to their order)
    sw = tab.clone()
    sw[b, 0], sw[b, 1] = tab[b, 1], tab[b, 0]
    out_sw, _, _ = run_decode(emu, kind, True, qkv, pool, sw, N, POS, cos, sin, hq, hkv, dtype, gs)
    assert not torch.equal(out_sw[b], out[b])


# ------------------------------------------------------------------------------------------------------------------ prefill
L_PRE = 256
# (pos0, n_tok): spans across the page edges 64, 128 and 192, a span starting on an edge, a span ending on one, an empty slot
PRE_CONFIGS = [([60, 0, 64, 127], [8, 0, 1, 3]), ([62, 190], [2, 3])]


def pre_data(gen, n_tok, hq, hkv, dtype):
    M = sum(n_tok)
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    return {"q": rn(M, hq * R.HD), "k": rn(M, hkv * R.HD), "v": rn(M, hkv * R.HD)}


def prefill_table(gen, pos0, n_tok):
    """Slots own pages through their last written row; only full pages below pos0 are shared."""
    ends = [p + n for p, n in zip(pos0, n_tok)]
    tab, N = scrambled_table(gen, ends, L_PRE // PG, shared=False)
    for b in range(1, len(pos0)):
        if pos0[b] >= PG and pos0[b - 1] >= PG:
            tab[b, 0] = tab[b - 1, 0]
    return tab, N


PREFILL_CASES = [("rows", None, F, G4), ("rows", None, BF, G8), ("rows", None, F, G1), ("rows_kv8", 64, F, G1), ("rows_kv8", 64, BF, G4),
                 ("rows_kv8", 128, F, G8), ("rows_kv8", 128, BF, G1), ("attn", None, F, G8), ("attn", None, BF, G1), ("attn", None, F, G4)]


@pytest.mark.parametrize("kind,gs,dtype,heads", PREFILL_CASES, ids=[f"{k}{gs or ''}-{DT_ID[d]}-G{h[0] // h[1]}" for k, gs, d, h in PREFILL_CASES])
def test_emulated_paged_prefill_equals_varlen_on_gathered_cache(emu, kind, gs, dtype, heads):
    """n_tok / pos0 straddling page edges (an empty slot included): q_out / attention rows, levels, meta and staging rows equal the
    _varlen kernel on the gathered cache bit for bit; nothing else in the pools changes; for the attention, swapping a slot's first and
    last page changes its output."""
    hq, hkv = heads
    gen = torch.Generator().manual_seed(31 * hq + hkv + CODE[dtype] + (gs or 0) + len(kind))
    cos, sin = R.tables(L_PRE, dtype, "cpu")
    code = CODE[dtype]
    for pos0, n_tok in PRE_CONFIGS:
        B = len(pos0)
        tab, N = prefill_table(gen, pos0, n_tok)
        pool = pools(gen, N, hkv, dtype, gs)
        d = pre_data(gen, n_tok, hq, hkv, dtype)
        flat = {n: gather(t, tab) for n, t in pool.items()}
        rows_of = [list(range(p, p + n)) for p, n in zip(pos0, n_tok)]
        head = [P(d["q"]), P(d["k"]), P(d["v"]), P(cos), P(sin)]
        qo, qo_ref = torch.zeros_like(d["q"]), torch.zeros_like(d["q"])
        if kind == "rows":
            pa, fa = {n: t.clone() for n, t in pool.items()}, {n: t.clone() for n, t in flat.items()}
            assert emu.hqq_b200_glue_rope_append_rows_paged(*head, P(pa["kc"]), P(pa["vc"]), P(tab), P(qo), ints(pos0), ints(n_tok), hq, hkv, L_PRE,
                                                            R.HD, B, N, code, None) == 0, emu.hqq_b200_last_error()
            assert emu.hqq_b200_glue_rope_append_rows_varlen(*head, P(fa["kc"]), P(fa["vc"]), P(qo_ref), ints(pos0), ints(n_tok), hq, hkv, L_PRE,
                                                             R.HD, B, code, None) == 0
            assert torch.equal(qo, qo_ref)
            check_pools(pool, pa, fa, tab, rows_of)
        elif kind == "rows_kv8":
            names = ("kq", "ks", "kz", "vq", "vs", "vz")
            pa, fa = {n: t.clone() for n, t in pool.items()}, {n: t.clone() for n, t in flat.items()}
            st = [torch.randn(B, hkv, L_PRE, R.HD, generator=gen).to(dtype) for _ in range(2)]
            sp, sf = [t.clone() for t in st], [t.clone() for t in st]
            assert emu.hqq_b200_glue_rope_append_rows_kv8_paged(*head, *[P(pa[n]) for n in names], P(tab), P(sp[0]), P(sp[1]), P(qo), ints(pos0),
                                                                ints(n_tok), hq, hkv, L_PRE, R.HD, gs, B, N, code, None) == 0, emu.hqq_b200_last_error()
            assert emu.hqq_b200_glue_rope_append_rows_kv8_varlen(*head, *[P(fa[n]) for n in names], P(sf[0]), P(sf[1]), P(qo_ref), ints(pos0),
                                                                 ints(n_tok), hq, hkv, L_PRE, R.HD, gs, B, code, None) == 0
            assert torch.equal(qo, qo_ref) and torch.equal(sp[0], sf[0]) and torch.equal(sp[1], sf[1])
            check_pools(pool, pa, fa, tab, rows_of)
        else:
            out, ref = torch.zeros_like(d["q"]), torch.zeros_like(d["q"])
            before = {n: t.clone() for n, t in pool.items()}
            assert emu.hqq_b200_glue_attn_prefill_paged(P(d["q"]), P(pool["kc"]), P(pool["vc"]), P(tab), P(out), ints(pos0), ints(n_tok), hq, hkv,
                                                        L_PRE, R.HD, B, N, code, None) == 0, emu.hqq_b200_last_error()
            assert emu.hqq_b200_glue_attn_prefill_varlen(P(d["q"]), P(flat["kc"]), P(flat["vc"]), P(ref), ints(pos0), ints(n_tok), hq, hkv, L_PRE,
                                                         R.HD, B, code, None) == 0
            assert torch.equal(out, ref)
            for n in pool:
                assert torch.equal(pool[n].view(torch.uint8), before[n].view(torch.uint8)), n
            b = max(range(B), key=lambda i: pos0[i] if n_tok[i] else -1)
            e = (pos0[b] + n_tok[b] - 1) // PG
            if e >= 1:  # its first page and its last, partly attended page trade places: the rows its first queries see change
                sw = tab.clone()
                sw[b, 0], sw[b, e] = tab[b, e], tab[b, 0]
                out_sw = torch.zeros_like(out)
                emu.hqq_b200_glue_attn_prefill_paged(P(d["q"]), P(pool["kc"]), P(pool["vc"]), P(sw), P(out_sw), ints(pos0), ints(n_tok), hq, hkv,
                                                     L_PRE, R.HD, B, N, code, None)
                r0 = sum(n_tok[:b])
                assert not torch.equal(out_sw[r0:r0 + n_tok[b]], out[r0:r0 + n_tok[b]])


@pytest.mark.parametrize("dtype,gs", [(F, 64), (BF, 128)], ids=["f16-gs64", "bf16-gs128"])
def test_emulated_kv8_stage_paged_equals_oracle_dequantize(emu, dtype, gs):
    """Staging rows [0, pos0[b]) of the slots in the chunk equal oracle.dequantize of the levels and meta gathered through the table;
    rows at or past pos0[b], and every row of a slot with n_tok 0, are untouched."""
    from oracle import hqq_oracle as o
    gen = torch.Generator().manual_seed(CODE[dtype] + gs)
    hkv = 2
    pos0, n_tok = [70, 64, 0, 63], [1, 5, 2, 0]  # rows across a page edge, up to one, none, a slot outside the chunk
    B = len(pos0)
    tab, N = prefill_table(gen, pos0, n_tok)
    pool = pools(gen, N, hkv, dtype, gs)
    names = ("kq", "ks", "kz", "vq", "vs", "vz")
    st = [torch.randn(B, hkv, L_PRE, R.HD, generator=gen).to(dtype) for _ in range(2)]
    st0 = [t.clone() for t in st]
    assert emu.hqq_b200_glue_kv8_stage_paged(*[P(pool[n]) for n in names], P(tab), P(st[0]), P(st[1]), ints(pos0), ints(n_tok), hkv, L_PRE, R.HD, gs, B,
                                             N, CODE[dtype], None) == 0, emu.hqq_b200_last_error()
    cdt = {torch.float16: "float16", torch.bfloat16: "bfloat16"}[dtype]
    for i, (lv, sc, ze) in enumerate((("kq", "ks", "kz"), ("vq", "vs", "vz"))):
        g = {n: gather(pool[n], tab) for n in (lv, sc, ze)}
        for b in range(B):
            p = pos0[b] if n_tok[b] else 0
            if p:
                meta = {"packing": None, "scale": g[sc][b, :, :p].float().reshape(-1, 1).numpy(), "zero": g[ze][b, :, :p].float().reshape(-1, 1).numpy(),
                        "shape": (hkv * p * R.HD // gs, gs), "nbits": 8}
                exp = o.dequantize(g[lv][b, :, :p].reshape(-1, gs).numpy(), meta, cdt).reshape(hkv, p, R.HD)
                assert np.array_equal(st[i][b, :, :p].float().numpy(), exp, equal_nan=True), (i, b)
            assert torch.equal(st[i][b, :, p:], st0[i][b, :, p:]), (i, b)


def test_emulated_paged_argument_checks(emu):
    """A null table, cache_len % 64 and n_pages < 1 are HQQ_E_INVALID for every _paged entry point, with its name in the message."""
    buf = torch.zeros(1 << 20, dtype=torch.uint8)
    b = P(buf)
    one, zero = ints([0]), ints([1])

    def calls(table, L, n):
        return {
            b"decode_batch_paged": lambda: emu.hqq_b200_glue_rope_attn_decode_batch_paged(*[b] * 7, table, b, b, 8, 2, L, R.HD, 1, n, F16, None),
            b"decode_split_paged": lambda: emu.hqq_b200_glue_rope_attn_decode_split_paged(*[b] * 7, table, b, b, b, 8, 2, L, R.HD, 1, n, F16, None),
            b"split_kv8_paged": lambda: emu.hqq_b200_glue_rope_attn_decode_split_kv8_paged(*[b] * 11, table, b, b, b, 8, 2, L, R.HD, 64, 1, n, F16, None),
            b"append_rows_paged": lambda: emu.hqq_b200_glue_rope_append_rows_paged(*[b] * 7, table, b, one, zero, 8, 2, L, R.HD, 1, n, F16, None),
            b"rows_kv8_paged": lambda: emu.hqq_b200_glue_rope_append_rows_kv8_paged(*[b] * 11, table, b, b, b, one, zero, 8, 2, L, R.HD, 64, 1, n, F16,
                                                                                     None),
            b"kv8_stage_paged": lambda: emu.hqq_b200_glue_kv8_stage_paged(*[b] * 6, table, b, b, one, zero, 2, L, R.HD, 64, 1, n, F16, None),
            b"attn_prefill_paged": lambda: emu.hqq_b200_glue_attn_prefill_paged(*[b] * 3, table, b, one, zero, 8, 2, L, R.HD, 1, n, F16, None),
        }
    for table, L, n in ((None, 128, 1), (b, 100, 1), (b, 128, 0), (b, 128, -3)):
        for name, fn in calls(table, L, n).items():
            assert fn() == E_INVALID, (name, table, L, n)
            assert name in emu.hqq_b200_last_error()


# ------------------------------------------------------------------------------------------------------------------ allocator
def conserved(a: PageAllocator):
    """Refcounts equal the table's references, free + held = N, and every entry lies in [0, N]."""
    refs = [0] * a.n_pages
    for row in a.table:
        for p in row:
            assert 0 <= p <= a.n_pages
            if p != a.sink:
                refs[p] += 1
    assert refs == a.ref
    assert sorted(a.free) == [p for p in range(a.n_pages) if refs[p] == 0]
    assert len(set(a.free)) == len(a.free)


def state(a):
    return ([r[:] for r in a.table], a.ref[:], sorted(a.free), a.pos[:], a.active[:])


def test_allocator_pages_follow_positions_and_wrap():
    a = PageAllocator(8, 2, 256)
    for step in range(256 + 70):
        a.step()
        conserved(a)
        p = step % 256  # the row this step wrote
        assert a.table[0][p // 64] != a.sink
        assert a.pages_of(0) == p // 64 + 1, step  # at the wrap the previous lap's pages went back first
        assert all(x == a.sink for x in a.table[0][p // 64 + 1:])
    assert a.pos == [70, 70]


def test_allocator_release_and_refill():
    a = PageAllocator(10, 3, 512)
    a.prefill({0: (0, 300), 1: (0, 65), 2: (0, 1)})
    conserved(a)
    assert [a.pages_of(b) for b in range(3)] == [5, 2, 1] and a.free_pages == 2
    a.release(0)
    conserved(a)
    assert a.free_pages == 7 and a.table[0] == [a.sink] * 8 and not a.active[0]
    for _ in range(64):  # a released slot gets no pages while it steps
        a.step()
    assert a.pages_of(0) == 0
    with pytest.raises(ValueError):  # positions [0, 10) of the released slot hold no pages
        a.prefill({0: (10, 5)})
    a.prefill({0: (0, 10)})
    assert a.active[0] and a.pages_of(0) == 1 and a.pos[0] == 10
    a.prefill({1: (0, 3)})  # a shorter refill returns the pages past its end
    assert a.pages_of(1) == 1
    conserved(a)


@pytest.mark.parametrize("p", [63, 64, 65])
def test_allocator_fork(p):
    a = PageAllocator(16, 4, 512)
    a.prefill({0: (0, p)})
    base = a.pages_of(0)
    for d in (1, 2, 3):
        _, copies = a.fork(0, d)
        assert a.pos[d] == p
        assert a.table[d][:p // 64] == a.table[0][:p // 64]
        assert len(copies) == (1 if p % 64 else 0)
        if p % 64:
            assert a.table[d][p // 64] != a.table[0][p // 64] and copies[0] == (a.table[0][p // 64], a.table[d][p // 64])
        conserved(a)
    assert 16 - a.free_pages == base + 3 * (1 if p % 64 else 0)
    w, _ = a.step()  # every slot writes row p: into its own page
    held = [a.table[b][p // 64] for b in range(4)]
    assert len(set(held)) == 4 and all(a.ref[x] == 1 for x in held)
    conserved(a)


def test_allocator_copy_on_write_into_shared_partial_page():
    a = PageAllocator(16, 2, 512)
    a.prefill({0: (0, 150)})
    a.fork(0, 1)
    shared = a.table[0][1]
    assert a.ref[shared] == 2
    w, copies = a.prefill({1: (100, 20)})  # enters shared page 1 mid-page: copied first
    assert copies and copies[0][0] == shared and a.table[1][1] == copies[0][1] != shared
    assert a.ref[shared] == 1 and a.table[0][1] == shared
    assert a.table[1][2] == a.sink  # past the refill's end
    conserved(a)


def test_allocator_out_of_pages_changes_nothing():
    a = PageAllocator(4, 3, 512)
    a.prefill({0: (0, 130)})
    a.fork(0, 1)
    s0 = state(a)
    with pytest.raises(RuntimeError):
        a.prefill({2: (0, 200)})
    assert state(a) == s0
    with pytest.raises(RuntimeError):
        a.fork(0, 2)  # needs a copy of the partial page: none left
    assert state(a) == s0
    a.release(1)  # its copied partial page comes back
    a.prefill({2: (0, 64)})  # and goes to slot 2, which now sits at a page edge
    s1 = state(a)
    with pytest.raises(RuntimeError):
        a.step()  # slot 2 needs a page, none is free
    assert state(a) == s1
    conserved(a)


def test_allocator_rejects_bad_options():
    for n, L in ((0, 256), (-1, 256), (4, 100), (2.5, 256)):
        with pytest.raises(ValueError):
            PageAllocator(n, 2, L)
