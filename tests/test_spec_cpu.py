"""Speculative decoding on the CPU kernel emulator (csrc/decode_glue.cu: the DEVPOS rows kernels, the verify attention, the n-gram
draft and accept kernels) and the page allocator's window / advance (harness.PageAllocator).

The verify attention is held element by element to a float64 attention over the cache within spec_ref's per-column bound, and four
planted defects must each leave that bound.  The paged forms equal the unpaged ones on the gathered cache bit for bit; the DEVPOS
append equals the _varlen append called with pos0 = pos bit for bit.  Lookup and accept equal spec_ref.py exactly."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import attn_split_ref as R  # noqa: E402
import spec_ref  # noqa: E402
from hqq_b200.harness import KV_PAGE, PageAllocator, kv8_dequantize  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
SMS = 4
E_INVALID = -1
VP, I = ctypes.c_void_p, ctypes.c_int
F, BF = torch.float16, torch.bfloat16
DT_ID = {F: "f16", BF: "bf16"}
L = 192


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    sig = {"hqq_b200_glue_rope_append_rows_devpos": [VP] * 9 + [I] * 7, "hqq_b200_glue_rope_append_rows_devpos_paged": [VP] * 10 + [I] * 8,
           "hqq_b200_glue_rope_append_rows_varlen": [VP] * 10 + [I] * 6, "hqq_b200_glue_attn_verify_split": [VP] * 6 + [I] * 7,
           "hqq_b200_glue_attn_verify_split_paged": [VP] * 7 + [I] * 8, "hqq_b200_glue_ngram_draft": [VP] * 4 + [I] * 3,
           "hqq_b200_glue_spec_accept": [VP] * 8 + [I] * 3, "hqq_b200_glue_rope_append_rows_kv8_devpos": [VP] * 13 + [I] * 8,
           "hqq_b200_glue_rope_append_rows_kv8_devpos_paged": [VP] * 14 + [I] * 9, "hqq_b200_glue_rope_append_rows_kv8_varlen": [VP] * 16 + [I] * 7,
           "hqq_b200_glue_attn_verify_split_kv8": [VP] * 10 + [I] * 8, "hqq_b200_glue_attn_verify_split_kv8_paged": [VP] * 11 + [I] * 9}
    for n, a in sig.items():
        getattr(lib, n).argtypes = a + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def n_groups(hq, hkv, T):
    return -(-T * (hq // hkv) // 16)


def ws_bytes(hq, hkv, T, B):
    g = B * hkv * n_groups(hq, hkv, T)
    return g * max(1, SMS // hkv) * 16 * 130 * 4 + g * 4


def page_table(gen, B):
    """A scrambled table [B, L / 64] over exactly B L / 64 pages (physical order differs from logical order)."""
    E = L // KV_PAGE
    perm = torch.randperm(B * E, generator=gen)
    return perm.view(B, E).to(torch.int32).contiguous(), B * E


def to_pool(cache, tab, N):
    """The pool [N + 1, hkv, 64, X] holding the contiguous cache [B, hkv, L, X] through tab; the sink NaN (levels 0xFF)."""
    B, hkv, _, hd = cache.shape
    pool = torch.full((N + 1, hkv, KV_PAGE, hd), 255 if cache.dtype == torch.uint8 else float("nan"), dtype=cache.dtype)
    for b in range(B):
        for j in range(L // KV_PAGE):
            pool[int(tab[b, j])] = cache[b, :, j * KV_PAGE:(j + 1) * KV_PAGE]
    return pool


def gather(pool, tab):
    B, E = tab.shape
    return pool[tab.long()].permute(0, 2, 1, 3, 4).reshape(B, pool.shape[1], E * KV_PAGE, pool.shape[3]).contiguous()


def run_verify(emu, q, kc, vc, pos, T, hq, hkv, dtype, tab=None, N=0):
    B = len(pos)
    out = torch.zeros(B * T, hq * R.HD, dtype=dtype)
    ws = torch.zeros(ws_bytes(hq, hkv, T, B), dtype=torch.uint8)
    p = torch.tensor(pos, dtype=torch.int64)
    if tab is None:
        rc = emu.hqq_b200_glue_attn_verify_split(P(q), P(kc), P(vc), P(p), P(out), P(ws), hq, hkv, L, R.HD, T, B, CODE[dtype], None)
    else:
        rc = emu.hqq_b200_glue_attn_verify_split_paged(P(q), P(kc), P(vc), P(tab), P(p), P(out), P(ws), hq, hkv, L, R.HD, T, B, N, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, ws[-4 * B * hkv * n_groups(hq, hkv, T):]


KV8_NAMES = ("kq", "ks", "kz", "vq", "vs", "vz")


def kv8_cache(gen, B, hkv, gs, dtype):
    """Random 8-bit caches: levels, scales and zeros in the range kv8_quantize_rows produces."""
    ng = R.HD // gs
    c = {n: torch.randint(0, 256, (B, hkv, L, R.HD), generator=gen, dtype=torch.uint8) for n in ("kq", "vq")}
    for n in ("ks", "vs"):
        c[n] = (torch.rand(B, hkv, L, ng, generator=gen) * 0.02 + 0.005).to(dtype)
    for n in ("kz", "vz"):
        c[n] = (torch.rand(B, hkv, L, ng, generator=gen) * 255).to(dtype)
    return c


def run_verify_kv8(emu, q, c, pos, T, hq, hkv, gs, dtype, tab=None, N=0):
    B = len(pos)
    out = torch.zeros(B * T, hq * R.HD, dtype=dtype)
    ws = torch.zeros(ws_bytes(hq, hkv, T, B), dtype=torch.uint8)
    p = torch.tensor(pos, dtype=torch.int64)
    cs = [P(c[n]) for n in KV8_NAMES]
    if tab is None:
        rc = emu.hqq_b200_glue_attn_verify_split_kv8(P(q), *cs, P(p), P(out), P(ws), hq, hkv, L, R.HD, gs, T, B, CODE[dtype], None)
    else:
        rc = emu.hqq_b200_glue_attn_verify_split_kv8_paged(P(q), *cs, P(tab), P(p), P(out), P(ws), hq, hkv, L, R.HD, gs, T, B, N, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, ws[-4 * B * hkv * n_groups(hq, hkv, T):]


KV8_CASES = [(F, (8, 2), 4, 64), (BF, (8, 1), 8, 64), (F, (2, 2), 2, 128), (BF, (8, 2), 8, 128)]


@pytest.mark.parametrize("dtype,heads,T,gs", KV8_CASES, ids=[f"{DT_ID[d]}-G{h[0] // h[1]}-T{t}-gs{g}" for d, h, t, g in KV8_CASES])
def test_emulated_verify_attention_kv8_within_bound_and_paged_equal(emu, dtype, heads, T, gs):
    """The 8-bit form: within the bound against float64 attention over the dequantised cache (kv8_dequantize), tickets at zero, the
    paged twin equal bit for bit."""
    hq, hkv = heads
    gen = torch.Generator().manual_seed(300 + 10 * hq + T + gs + CODE[dtype])
    S = R.split_count(SMS, hkv, L)
    for pos in ([0, 17, 64], [95, L - T, L - 2]):
        B = len(pos)
        q = torch.randn(B * T, hq * R.HD, generator=gen).to(dtype)
        c = kv8_cache(gen, B, hkv, gs, dtype)
        out, tk = run_verify_kv8(emu, q, c, pos, T, hq, hkv, gs, dtype)
        assert torch.count_nonzero(tk) == 0
        kc, vc = kv8_dequantize(c["kq"], c["ks"], c["kz"]), kv8_dequantize(c["vq"], c["vs"], c["vz"])
        y, bound = spec_ref.verify_reference(q, kc, vc, pos, T, dtype, S)
        rows = valid_rows(pos, T)
        ratio, ok = R.within(out[rows], y[rows], bound[rows])
        assert ok, f"pos {pos}: error / bound {ratio:.3f}"
        tab, N = page_table(gen, B)
        outp, tkp = run_verify_kv8(emu, q, {n: to_pool(t, tab, N) for n, t in c.items()}, pos, T, hq, hkv, gs, dtype, tab, N)
        assert torch.equal(outp[rows], out[rows]) and torch.count_nonzero(tkp) == 0


@pytest.mark.parametrize("dtype,gs", [(F, 64), (BF, 128)], ids=["f16-gs64", "bf16-gs128"])
def test_emulated_kv8_devpos_append_equals_varlen(emu, dtype, gs):
    """The 8-bit DEVPOS append writes the levels and meta of the _varlen kv8 append (pos0 = pos) bit for bit, no staging rows, and
    rows t >= n[b] are neither written nor rotated; the paged twin writes the same rows through a scrambled table."""
    hq, hkv, T = 8, 2, 4
    gen = torch.Generator().manual_seed(21 + gs + CODE[dtype])
    pos = [0, 63, L - 2]
    B = len(pos)
    q, k, v = rows_inputs(gen, B, T, hq, hkv, dtype)
    cos, sin = R.tables(L, dtype, "cpu")
    c0 = kv8_cache(gen, B, hkv, gs, dtype)
    p = torch.tensor(pos, dtype=torch.int64)
    c = {n: t.clone() for n, t in c0.items()}
    qo = torch.full((B * T, hq * R.HD), 7.0, dtype=dtype)
    assert emu.hqq_b200_glue_rope_append_rows_kv8_devpos(P(q), P(k), P(v), P(cos), P(sin), *[P(c[n]) for n in KV8_NAMES], P(qo), P(p), T, hq, hkv, L,
                                                          R.HD, gs, B, CODE[dtype], None) == 0
    n = [min(T, L - x) for x in pos]
    rows = valid_rows(pos, T)
    cv = {nm: t.clone() for nm, t in c0.items()}
    st = [torch.zeros(B, hkv, L, R.HD, dtype=dtype) for _ in range(2)]
    qv = torch.zeros(len(rows), hq * R.HD, dtype=dtype)
    ints = lambda xs: (ctypes.c_int * len(xs))(*xs)
    assert emu.hqq_b200_glue_rope_append_rows_kv8_varlen(P(q[rows].contiguous()), P(k[rows].contiguous()), P(v[rows].contiguous()), P(cos), P(sin),
                                                          *[P(cv[nm]) for nm in KV8_NAMES], P(st[0]), P(st[1]), P(qv), ints(pos), ints(n), hq, hkv, L,
                                                          R.HD, gs, B, CODE[dtype], None) == 0
    for nm in KV8_NAMES:
        assert torch.equal(c[nm], cv[nm]), nm
    assert torch.equal(qo[rows], qv)
    skipped = [r for r in range(B * T) if r not in rows]
    assert skipped and bool((qo[skipped] == 7.0).all())
    tab, N = page_table(gen, B)
    pools = {nm: to_pool(t, tab, N) for nm, t in c0.items()}
    qp = torch.zeros_like(qo)
    assert emu.hqq_b200_glue_rope_append_rows_kv8_devpos_paged(P(q), P(k), P(v), P(cos), P(sin), *[P(pools[nm]) for nm in KV8_NAMES], P(tab), P(qp),
                                                                P(p), T, hq, hkv, L, R.HD, gs, B, N, CODE[dtype], None) == 0
    for nm in KV8_NAMES:
        assert torch.equal(gather(pools[nm], tab), c[nm]), nm
    assert torch.equal(qp[rows], qo[rows])


def valid_rows(pos, T):
    return [b * T + t for b in range(len(pos)) for t in range(min(T, L - pos[b]))]


# positions: 0, 15, 16, 17, 63, 64, a split-chunk edge (S = 2 at n_kv = 2: chunks of 96 at end 192), cache_len - T, cache_len - 2
POS_SETS = [[0, 15, 16], [17, 63, 64], [95, L - 8, L - 2]]
VER_CASES = [(F, (2, 2), 1), (BF, (2, 2), 4), (F, (8, 2), 2), (BF, (8, 2), 8), (F, (8, 1), 4), (BF, (8, 1), 8), (F, (8, 2), 8), (BF, (8, 1), 1)]


@pytest.mark.parametrize("dtype,heads,T", VER_CASES, ids=[f"{DT_ID[d]}-G{h[0] // h[1]}-T{t}" for d, h, t in VER_CASES])
def test_emulated_verify_attention_within_bound_and_paged_equal(emu, dtype, heads, T):
    """Every valid output element within spec_ref's float64 bound, tickets back at zero, the paged twin equal bit for bit on a
    scrambled table."""
    hq, hkv = heads
    gen = torch.Generator().manual_seed(100 * hq + 10 * hkv + T + CODE[dtype])
    S = R.split_count(SMS, hkv, L)
    for pos in POS_SETS:
        B = len(pos)
        q = torch.randn(B * T, hq * R.HD, generator=gen).to(dtype)
        kc = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
        vc = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
        out, tk = run_verify(emu, q, kc, vc, pos, T, hq, hkv, dtype)
        assert torch.count_nonzero(tk) == 0
        y, bound = spec_ref.verify_reference(q, kc, vc, pos, T, dtype, S)
        rows = valid_rows(pos, T)
        ratio, ok = R.within(out[rows], y[rows], bound[rows])
        assert ok, f"pos {pos}: error / bound {ratio:.3f}"
        assert torch.isfinite(out.float()).all()
        tab, N = page_table(gen, B)
        outp, tkp = run_verify(emu, q, to_pool(kc, tab, N), to_pool(vc, tab, N), pos, T, hq, hkv, dtype, tab, N)
        assert torch.equal(outp[rows], out[rows]) and torch.count_nonzero(tkp) == 0


def test_emulated_verify_attention_planted_defects_leave_the_bound(emu):
    """The mask off by one, the draft rows dropped, the column -> head mapping transposed and a dropped split each leave the bound."""
    hq, hkv, T, dtype = 8, 2, 4, F
    gen = torch.Generator().manual_seed(5)
    S = R.split_count(SMS, hkv, L)
    pos = [40, 100, 150]
    B = len(pos)
    q = torch.randn(B * T, hq * R.HD, generator=gen).to(dtype)
    kc = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
    vc = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
    y, bound = spec_ref.verify_reference(q, kc, vc, pos, T, dtype, S)
    rows = valid_rows(pos, T)
    out, _ = run_verify(emu, q, kc, vc, pos, T, hq, hkv, dtype)
    assert R.within(out[rows], y[rows], bound[rows])[1]
    for k, bad in enumerate(spec_ref.verify_defects(q, kc, vc, pos, T)):
        bad = bad[rows]
        m = torch.isfinite(bad)
        assert m.any()
        assert ((bad[m] - y[rows][m]).abs() > bound[rows][m]).any(), f"defect {k} stays inside the bound"


def rows_inputs(gen, B, T, hq, hkv, dtype):
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    return rn(B * T, hq * R.HD), rn(B * T, hkv * R.HD), rn(B * T, hkv * R.HD)


@pytest.mark.parametrize("dtype", [F, BF], ids=["f16", "bf16"])
def test_emulated_devpos_append_equals_varlen(emu, dtype):
    """DEVPOS rows equal the _varlen rows (pos0 = pos, n_tok = n) bit for bit, rows t >= n[b] are neither written nor rotated, and
    the paged twin writes the same rows through a scrambled table."""
    hq, hkv, T = 8, 2, 8
    gen = torch.Generator().manual_seed(11 + CODE[dtype])
    pos = [0, 63, L - 3, 100]
    B = len(pos)
    q, k, v = rows_inputs(gen, B, T, hq, hkv, dtype)
    cos, sin = R.tables(L, dtype, "cpu")
    kc0 = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
    vc0 = torch.randn(B, hkv, L, R.HD, generator=gen).to(dtype)
    p = torch.tensor(pos, dtype=torch.int64)
    kc, vc = kc0.clone(), vc0.clone()
    qo = torch.full((B * T, hq * R.HD), 7.0, dtype=dtype)
    assert emu.hqq_b200_glue_rope_append_rows_devpos(P(q), P(k), P(v), P(cos), P(sin), P(kc), P(vc), P(qo), P(p), T, hq, hkv, L, R.HD, B, CODE[dtype],
                                                      None) == 0
    n = [min(T, L - x) for x in pos]
    rows = valid_rows(pos, T)
    kv_, vv_ = kc0.clone(), vc0.clone()
    qv = torch.zeros(len(rows), hq * R.HD, dtype=dtype)
    ints = lambda xs: (ctypes.c_int * len(xs))(*xs)
    assert emu.hqq_b200_glue_rope_append_rows_varlen(P(q[rows].contiguous()), P(k[rows].contiguous()), P(v[rows].contiguous()), P(cos), P(sin), P(kv_),
                                                      P(vv_), P(qv), ints(pos), ints(n), hq, hkv, L, R.HD, B, CODE[dtype], None) == 0
    assert torch.equal(kc, kv_) and torch.equal(vc, vv_)
    assert torch.equal(qo[rows], qv)
    skipped = [r for r in range(B * T) if r not in rows]
    assert skipped and bool((qo[skipped] == 7.0).all())
    tab, N = page_table(gen, B)
    kp, vp = to_pool(kc0, tab, N), to_pool(vc0, tab, N)
    qp = torch.zeros_like(qo)
    assert emu.hqq_b200_glue_rope_append_rows_devpos_paged(P(q), P(k), P(v), P(cos), P(sin), P(kp), P(vp), P(tab), P(qp), P(p), T, hq, hkv, L, R.HD, B,
                                                            N, CODE[dtype], None) == 0
    assert torch.equal(gather(kp, tab), kc) and torch.equal(gather(vp, tab), vc) and torch.equal(qp[rows], qo[rows])


def run_ngram(emu, hist, pos, tok, K):
    B = len(pos)
    h = torch.tensor(hist, dtype=torch.int32)
    d = torch.zeros(B, K, dtype=torch.int64)
    assert emu.hqq_b200_glue_ngram_draft(P(h), P(torch.tensor(pos, dtype=torch.int64)), P(torch.tensor(tok, dtype=torch.int64)), P(d), h.shape[1], K, B,
                                         None) == 0
    return d.tolist()


def test_emulated_ngram_drafts_equal_spec_ref(emu):
    """No match, several matches (the latest wins), a longer n preferred, truncation at L, L < n, and random histories."""
    Lh, K = 64, 5
    cases = [  # (history before pos, tok)
        ([1, 2, 3, 4, 5], 9),                     # no match
        ([7, 1, 2, 7, 3, 4, 7, 5], 7),            # several 1-gram matches: the latest (j = 6) wins
        ([1, 2, 9, 8, 2, 9, 5, 1, 2, 6, 1], 2),   # 2-gram "1 2" at j = 0 and 7 preferred to later 1-gram matches
        ([4, 5, 6, 1, 4, 5], 6),                  # 3-gram, drafts truncated at L
        ([3], 3),                                 # L = 2 < 3: only the 1-gram
        ([], 5),                                  # L = 1: nothing
        ([5, 5, 5, 5], 5),                        # overlapping matches
    ]
    gen = torch.Generator().manual_seed(3)
    for _ in range(6):
        n = int(torch.randint(1, Lh - 1, (1,), generator=gen))
        seq = torch.randint(0, 4, (n + 1,), generator=gen).tolist()
        cases.append((seq[:n], seq[n]))
    hist = [[0] * Lh for _ in cases]
    for b, (h, _) in enumerate(cases):
        hist[b][:len(h)] = h
        hist[b][len(h)] = 99  # hist[pos] is not read: tok stands for it
    got = run_ngram(emu, hist, [len(h) for h, _ in cases], [t for _, t in cases], K)
    for b, (h, t) in enumerate(cases):
        assert got[b] == spec_ref.ngram_drafts(h, len(h), t, K), (b, h, t)


def test_emulated_accept_equals_spec_ref(emu):
    """All / none / partial acceptance, sentinels, and a clamped window that wraps pos to 0."""
    K, Lh = 4, 32
    T = K + 1
    slots = [  # (pos, tok, drafts, targets)
        (3, 10, [1, 2, 3, 4], [1, 2, 3, 4, 5]),     # all accepted
        (5, 11, [1, 2, 3, 4], [9, 2, 3, 4, 5]),     # none
        (7, 12, [1, 2, 3, 4], [1, 2, 8, 4, 5]),     # partial: a = 2
        (9, 13, [1, -1, 3, 4], [1, 2, 3, 4, 5]),    # sentinel stops at 1
        (Lh - 3, 14, [1, 2, 3, 4], [1, 2, 3, 4, 5]),  # n = 3: a = 2, pos wraps to 0
        (Lh - 1, 15, [1, 2, 3, 4], [1, 2, 3, 4, 5]),  # n = 1: only t_0
    ]
    B = len(slots)
    pos = torch.tensor([s[0] for s in slots], dtype=torch.int64)
    tok = torch.tensor([s[1] for s in slots], dtype=torch.int64)
    nxt = torch.zeros(B, dtype=torch.int64)
    d = torch.tensor([s[2] for s in slots], dtype=torch.int64)
    tg = torch.tensor([s[3] for s in slots], dtype=torch.int64)
    hist = torch.full((B, Lh), -5, dtype=torch.int32)
    out = torch.zeros(B, T, dtype=torch.int64)
    n_new = torch.zeros(B, dtype=torch.int64)
    assert emu.hqq_b200_glue_spec_accept(P(tg), P(d), P(pos), P(tok), P(nxt), P(hist), P(out), P(n_new), Lh, K, B, None) == 0
    for b, (p, t, dr, tr) in enumerate(slots):
        em, a, np_ = spec_ref.accept(t, dr, tr, p, Lh)
        assert out[b].tolist() == em + [-1] * (T - len(em))
        assert int(n_new[b]) == a + 1 and int(pos[b]) == np_
        assert int(tok[b]) == int(nxt[b]) == tr[a]
        want = [-5] * Lh
        for i, x in enumerate([t] + dr[:a]):
            want[p + i] = x
        assert hist[b].tolist() == want
    assert int(pos[4]) == 0


def test_emulated_spec_entry_points_reject_bad_arguments(emu):
    z = torch.zeros(1 << 16, dtype=torch.uint8)
    p = torch.zeros(4, dtype=torch.int64)
    for T in (0, 9):
        assert emu.hqq_b200_glue_attn_verify_split(P(z), P(z), P(z), P(p), P(z), P(z), 8, 2, L, 128, T, 1, F16, None) == E_INVALID
        assert emu.hqq_b200_glue_rope_append_rows_devpos(P(z), P(z), P(z), P(z), P(z), P(z), P(z), P(z), P(p), T, 8, 2, L, 128, 1, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_attn_verify_split(P(z), P(z), P(z), None, P(z), P(z), 8, 2, L, 128, 2, 1, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_attn_verify_split_paged(P(z), P(z), P(z), None, P(p), P(z), P(z), 8, 2, L, 128, 2, 1, 3, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_attn_verify_split_paged(P(z), P(z), P(z), P(z), P(p), P(z), P(z), 8, 2, 100, 128, 2, 1, 3, F16, None) == E_INVALID
    for K in (0, 8):
        assert emu.hqq_b200_glue_ngram_draft(P(z), P(p), P(p), P(z), L, K, 1, None) == E_INVALID
        assert emu.hqq_b200_glue_spec_accept(P(z), P(z), P(p), P(p), P(p), P(z), P(z), P(z), L, K, 1, None) == E_INVALID
    assert emu.hqq_b200_glue_ngram_draft(P(z), P(p), P(p), P(z), 0, 2, 1, None) == E_INVALID
    assert emu.hqq_b200_glue_spec_accept(P(z), P(z), P(p), P(p), P(p), P(z), P(z), P(z), L, 2, 0, None) == E_INVALID


# ------------------------------------------------------------------------------------------------------------------ allocator
def check_invariant(pa):
    """Entries past the page of each active slot's last written row are the sink; refcounts match the table; the free list and
    the held pages partition the pool."""
    held = {}
    for b in range(pa.batch):
        for j, p in enumerate(pa.table[b]):
            if p != pa.sink:
                held[p] = held.get(p, 0) + 1
        first_free = -(-pa.pos[b] // KV_PAGE)
        if pa.active[b]:
            assert all(pa.table[b][j] == pa.sink for j in range(first_free, pa.entries)), (b, pa.pos[b], pa.table[b])
    assert all(pa.ref[p] == c for p, c in held.items())
    assert sorted(list(held) + pa.free) == list(range(pa.n_pages))


def test_allocator_spec_window_and_advance():
    """Conservation and the invariant across windows, advances, a wrap, and fork plus spec."""
    Lc, K = 256, 7
    pa = PageAllocator(12, 3, Lc)
    pa.prefill({0: (0, 60), 1: (0, 64), 2: (0, 1)})
    check_invariant(pa)
    w, _ = pa.spec_window(K)  # slot 0: rows 60 .. 67 enter entry 1 at row 64; slot 1 enters entry 1 at its first row
    assert {(b, j) for b, j, p in w if p != pa.sink} == {(0, 1), (1, 1)}
    pa.spec_advance([2, 8, 1])  # slot 0 stays inside entry 0: entry 1 goes back
    check_invariant(pa)
    assert pa.pos == [62, 72, 2] and pa.table[0][1] == pa.sink and pa.table[1][1] != pa.sink
    pa.fork(1, 2)
    check_invariant(pa)
    shared = pa.table[1][0]
    assert pa.table[2][0] == shared and pa.ref[shared] == 2
    pa.spec_window(K)
    assert pa.table[2][0] == shared  # a shared page is never written: windows start past it
    pa.spec_advance([8, 8, 8])
    check_invariant(pa)
    for b in range(3):  # walk every slot to the cache end: the window clamps, the advance wraps to 0 and returns the lap
        while pa.pos[b] != 0:
            pa.spec_window(K)
            pa.spec_advance([min(K + 1, Lc - p) if i == b else 0 for i, p in enumerate(pa.pos)])
            check_invariant(pa)
    assert pa.free_pages == pa.n_pages
    w, _ = pa.spec_window(K)  # at 0 after the wrap: fresh pages again
    assert sum(p != pa.sink for _, _, p in w) == 3


def test_allocator_spec_window_out_of_pages_changes_nothing():
    """Two slots that both enter a new page, one free page: spec_window raises RuntimeError and leaves table, refcounts, free list,
    positions and active slots exactly as they were just before the call."""
    pa = PageAllocator(3, 2, 256)
    pa.prefill({0: (0, 60), 1: (0, 64)})
    assert pa.free_pages == 1
    snap = ([r[:] for r in pa.table], pa.ref[:], pa.free[:], pa.pos[:], pa.active[:])
    with pytest.raises(RuntimeError):
        pa.spec_window(7)
    assert ([r[:] for r in pa.table], pa.ref, pa.free, pa.pos, pa.active) == snap
    check_invariant(pa)
    pa.release(1)  # with slot 1's page back, the same window fits
    w, _ = pa.spec_window(7)
    assert [(b, j) for b, j, p in w if p != pa.sink] == [(0, 1)]
    pa.spec_advance([8, 1])
    check_invariant(pa)
