"""Ragged batches on the CPU kernel emulator: the _seqpos decode attention entry points (one position per sequence) and the _varlen
prefill entry points (prompts of different lengths packed in slot order), csrc/decode_glue.cu.

Both are held bit for bit to the existing entry points called with batch 1 on each slot's slices: a sequence's output, cache rows
and tickets must not depend on which other sequences share its launch or where they sit.  The data separate the positions: every
sequence's batch-1 result at pos[0] differs from its result at pos[b], so a kernel that read pos[0] for every sequence fails."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
import attn_split_ref as R  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
SMS = 4
E_INVALID = -1
VP, I = ctypes.c_void_p, ctypes.c_int
HEADS = [(2, 2), (8, 2), (8, 1)]  # G = 1, 4, 8
DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    for n in ("hqq_b200_glue_rope_attn_decode_batch", "hqq_b200_glue_rope_attn_decode_batch_seqpos"):
        getattr(lib, n).argtypes = [VP] * 9 + [I] * 6 + [VP]
    for n in ("hqq_b200_glue_rope_attn_decode_split", "hqq_b200_glue_rope_attn_decode_split_seqpos"):
        getattr(lib, n).argtypes = [VP] * 10 + [I] * 6 + [VP]
    for n in ("hqq_b200_glue_rope_attn_decode_split_kv8", "hqq_b200_glue_rope_attn_decode_split_kv8_seqpos"):
        getattr(lib, n).argtypes = [VP] * 14 + [I] * 7 + [VP]
    lib.hqq_b200_glue_rope_append_rows.argtypes = [VP] * 8 + [I] * 8 + [VP]
    lib.hqq_b200_glue_rope_append_rows_varlen.argtypes = [VP] * 10 + [I] * 6 + [VP]
    lib.hqq_b200_glue_rope_append_rows_kv8.argtypes = [VP] * 14 + [I] * 9 + [VP]
    lib.hqq_b200_glue_rope_append_rows_kv8_varlen.argtypes = [VP] * 16 + [I] * 7 + [VP]
    lib.hqq_b200_glue_attn_prefill.argtypes = [VP] * 4 + [I] * 8 + [VP]
    lib.hqq_b200_glue_attn_prefill_varlen.argtypes = [VP] * 6 + [I] * 6 + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def ints(xs):
    return (ctypes.c_int * len(xs))(*xs)


# ------------------------------------------------------------------------------------------------------------------ decode
CACHE_NAMES = {"batch": ("kc", "vc"), "split": ("kc", "vc"), "kv8": ("kq", "ks", "kz", "vq", "vs", "vz")}


def decode_case(gen, kind, B, hq, hkv, L, dtype, gs):
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    c = {"q": rn(B, hq * R.HD), "k": rn(B, hkv * R.HD), "v": rn(B, hkv * R.HD)}
    if kind == "kv8":
        ng = R.HD // gs
        c["kq"] = torch.randint(0, 256, (B, hkv, L, R.HD), generator=gen, dtype=torch.uint8)
        c["vq"] = torch.randint(0, 256, (B, hkv, L, R.HD), generator=gen, dtype=torch.uint8)
        for n in ("ks", "vs"):
            c[n] = (torch.rand(B, hkv, L, ng, generator=gen) * 0.02 + 0.005).to(dtype)
        for n in ("kz", "vz"):
            c[n] = (torch.rand(B, hkv, L, ng, generator=gen) * 255).to(dtype)
    else:
        c["kc"], c["vc"] = rn(B, hkv, L, R.HD), rn(B, hkv, L, R.HD)
    return c


def run_decode(emu, kind, seqpos, case, pos, cos, sin, hq, hkv, dtype, gs):
    """One launch over case's batch at positions pos (a list: one element for the lock-step entry points); returns the output, the
    caches after the call and the tickets."""
    B, L = case["q"].shape[0], case[CACHE_NAMES[kind][0]].shape[2]
    c = {n: case[n].clone() for n in CACHE_NAMES[kind]}
    out = torch.zeros(B, hq * R.HD, dtype=dtype)
    p = torch.tensor(pos, dtype=torch.int64)
    ws = torch.zeros(R.workspace_bytes(SMS, hq, hkv, B), dtype=torch.uint8)
    sfx = "_seqpos" if seqpos else ""
    head = [P(case["q"]), P(case["k"]), P(case["v"]), P(cos), P(sin)]
    if kind == "batch":
        rc = getattr(emu, "hqq_b200_glue_rope_attn_decode_batch" + sfx)(*head, P(c["kc"]), P(c["vc"]), P(p), P(out), hq, hkv, L, R.HD, B, CODE[dtype], None)
    elif kind == "split":
        rc = getattr(emu, "hqq_b200_glue_rope_attn_decode_split" + sfx)(*head, P(c["kc"]), P(c["vc"]), P(p), P(out), P(ws), hq, hkv, L, R.HD, B,
                                                                       CODE[dtype], None)
    else:
        rc = getattr(emu, "hqq_b200_glue_rope_attn_decode_split_kv8" + sfx)(*head, *[P(c[n]) for n in CACHE_NAMES[kind]], P(p), P(out), P(ws), hq, hkv, L,
                                                                           R.HD, gs, B, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, c, ws[-4 * B * hkv:]


def slot(case, b, kind):
    return {n: t[b:b + 1].clone() for n, t in case.items()}


DECODE_KINDS = [("batch", 64), ("split", 64), ("kv8", 64), ("kv8", 128)]


@pytest.mark.parametrize("hq,hkv", HEADS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind,gs", DECODE_KINDS, ids=["batch", "split", "kv8_gs64", "kv8_gs128"])
def test_emulated_seqpos_decode_equals_batch1_per_sequence(emu, kind, gs, dtype, hq, hkv):
    """Each sequence of a _seqpos launch at mixed positions {0, 15, 16, 17, a split-chunk edge, cache_len - 1}: its output, its cache
    rows (all of them: row pos[b] written, the others untouched) and the tickets equal the lock-step entry point called with batch 1
    on its slices at pos[b], bit for bit; with all positions equal the launch equals the lock-step batched call."""
    L = 160
    S = R.split_count(SMS, hkv, L)
    edge = 32 * S - 1  # (edge + 1) / S is a whole number of 16-position tiles: the chunks end exactly at the last position
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(100 * hq + 10 * hkv + CODE[dtype] + gs + len(kind))
    for pos in ([0, 17, edge, L - 1], [16, L - 1, 15, 0], [edge, 0, 17]):
        B = len(pos)
        case = decode_case(gen, kind, B, hq, hkv, L, dtype, gs)
        out, c, tk = run_decode(emu, kind, True, case, pos, cos, sin, hq, hkv, dtype, gs)
        assert torch.count_nonzero(tk) == 0
        for b in range(B):
            one = slot(case, b, kind)
            o1, c1, tk1 = run_decode(emu, kind, False, one, [pos[b]], cos, sin, hq, hkv, dtype, gs)
            assert torch.equal(out[b:b + 1], o1), (pos, b)
            for n in CACHE_NAMES[kind]:
                assert torch.equal(c[n][b:b + 1], c1[n]), (pos, b, n)
            assert torch.count_nonzero(tk1) == 0
            if pos[b] != pos[0]:  # the data separate the positions: reading pos[0] would give another result
                o0, _, _ = run_decode(emu, kind, False, one, [pos[0]], cos, sin, hq, hkv, dtype, gs)
                assert not torch.equal(o0, o1), (pos, b)
    case = decode_case(gen, kind, 4, hq, hkv, L, dtype, gs)
    out, c, _ = run_decode(emu, kind, True, case, [17] * 4, cos, sin, hq, hkv, dtype, gs)
    out0, c0, _ = run_decode(emu, kind, False, case, [17], cos, sin, hq, hkv, dtype, gs)
    assert torch.equal(out, out0)
    for n in CACHE_NAMES[kind]:
        assert torch.equal(c[n], c0[n]), n


# ------------------------------------------------------------------------------------------------------------------ prefill
L_PRE = 1152
VARLEN_CONFIGS = [([17, 0, 130, 65], [1000, 63, 0, 64]), ([64, 1, 65], [63, 1000, 0])]


def varlen_data(gen, n_tok, hq, hkv, dtype, gs):
    B, M = len(n_tok), sum(n_tok)
    rn = lambda *s: torch.randn(*s, generator=gen).to(dtype)
    d = {"q": rn(M, hq * R.HD), "k": rn(M, hkv * R.HD), "v": rn(M, hkv * R.HD), "kc": rn(B, hkv, L_PRE, R.HD), "vc": rn(B, hkv, L_PRE, R.HD)}
    ng = R.HD // gs
    d["kq"] = torch.randint(0, 256, (B, hkv, L_PRE, R.HD), generator=gen, dtype=torch.uint8)
    d["vq"] = torch.randint(0, 256, (B, hkv, L_PRE, R.HD), generator=gen, dtype=torch.uint8)
    for n in ("ks", "kz", "vs", "vz"):
        d[n] = rn(B, hkv, L_PRE, ng)
    d["kst"], d["vst"] = rn(B, hkv, L_PRE, R.HD), rn(B, hkv, L_PRE, R.HD)
    return d


KV8 = ("kq", "ks", "kz", "vq", "vs", "vz", "kst", "vst")


def append(emu, kind, d, pos0, n_tok, cos, sin, hq, hkv, dtype, gs, varlen):
    """The rows kernel (kind "rows" or "rows_kv8") on d's slots; returns q_out and the caches after the call."""
    B, M = d["kc"].shape[0], d["q"].shape[0]
    qo = torch.zeros(M, hq * R.HD, dtype=dtype)
    head = [P(d["q"]), P(d["k"]), P(d["v"]), P(cos), P(sin)]
    if kind == "rows":
        c = {n: d[n].clone() for n in ("kc", "vc")}
        if varlen:
            rc = emu.hqq_b200_glue_rope_append_rows_varlen(*head, P(c["kc"]), P(c["vc"]), P(qo), ints(pos0), ints(n_tok), hq, hkv, L_PRE, R.HD, B,
                                                          CODE[dtype], None)
        else:
            rc = emu.hqq_b200_glue_rope_append_rows(*head, P(c["kc"]), P(c["vc"]), P(qo), pos0[0], n_tok[0], hq, hkv, L_PRE, R.HD, B, CODE[dtype], None)
    else:
        c = {n: d[n].clone() for n in KV8}
        ptrs = [P(c[n]) for n in KV8]
        if varlen:
            rc = emu.hqq_b200_glue_rope_append_rows_kv8_varlen(*head, *ptrs, P(qo), ints(pos0), ints(n_tok), hq, hkv, L_PRE, R.HD, gs, B, CODE[dtype], None)
        else:
            rc = emu.hqq_b200_glue_rope_append_rows_kv8(*head, *ptrs, P(qo), pos0[0], n_tok[0], hq, hkv, L_PRE, R.HD, gs, B, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return qo, c


def attn(emu, d, pos0, n_tok, hq, dtype, varlen):
    B, hkv, M = d["kc"].shape[0], d["kc"].shape[1], d["q"].shape[0]
    out = torch.zeros(M, hq * R.HD, dtype=dtype)
    if varlen:
        rc = emu.hqq_b200_glue_attn_prefill_varlen(P(d["q"]), P(d["kc"]), P(d["vc"]), P(out), ints(pos0), ints(n_tok), hq, hkv, L_PRE, R.HD, B,
                                                   CODE[dtype], None)
    else:
        rc = emu.hqq_b200_glue_attn_prefill(P(d["q"]), P(d["kc"]), P(d["vc"]), P(out), pos0[0], n_tok[0], hq, hkv, L_PRE, R.HD, B, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out


def slot_data(d, b, r0, n):
    """Slot b of d as a batch-1 problem: its n token rows from r0 and its caches."""
    return {k: (t[r0:r0 + n].clone() if k in ("q", "k", "v") else t[b:b + 1].clone()) for k, t in d.items()}


# the attention runs over 1130 cached positions, slow on the emulator: G = 1 and G = 8 only
VARLEN_CASES = [(k, gs, hq, hkv) for k, gs in (("rows", 64), ("rows_kv8", 64), ("rows_kv8", 128)) for hq, hkv in HEADS] + \
    [("attn", 64, hq, hkv) for hq, hkv in ((2, 2), (8, 1))]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind,gs,hq,hkv", VARLEN_CASES)
def test_emulated_varlen_prefill_equals_batch1_per_slot(emu, kind, gs, dtype, hq, hkv):
    """A _varlen launch with n_tok mixing {0, 1, 17, 64, 65, 130} and pos0 mixing {0, 63, 64, 1000}: q_out / attention rows, cache
    rows (levels, meta and staging rows for kv8) of every slot equal the fixed-length entry point called with batch 1 on that slot,
    bit for bit; a slot with no rows keeps its caches byte for byte; equal lengths give the fixed-length batched call."""
    cos, sin = R.tables(L_PRE, dtype, "cpu")
    gen = torch.Generator().manual_seed(1000 * hq + 10 * hkv + CODE[dtype] + gs + len(kind))
    for n_tok, pos0 in VARLEN_CONFIGS:
        d = varlen_data(gen, n_tok, hq, hkv, dtype, gs)
        if kind == "attn":
            got, caches = attn(emu, d, pos0, n_tok, hq, dtype, True), {}
        else:
            got, caches = append(emu, kind, d, pos0, n_tok, cos, sin, hq, hkv, dtype, gs, True)
        r0 = 0
        for b, (n, p0) in enumerate(zip(n_tok, pos0)):
            if n == 0:
                for k, t in caches.items():
                    assert torch.equal(t[b], d[k][b]), (b, k)
                continue
            one = slot_data(d, b, r0, n)
            if kind == "attn":
                exp, exp_c = attn(emu, one, [p0], [n], hq, dtype, False), {}
            else:
                exp, exp_c = append(emu, kind, one, [p0], [n], cos, sin, hq, hkv, dtype, gs, False)
            assert torch.equal(got[r0:r0 + n], exp), (n_tok, pos0, b)
            for k, t in exp_c.items():
                assert torch.equal(caches[k][b:b + 1], t), (n_tok, pos0, b, k)
            if p0 != pos0[0] and pos0[0] + n <= L_PRE:  # the data separate the positions
                alt = attn(emu, one, [pos0[0]], [n], hq, dtype, False) if kind == "attn" else \
                    append(emu, kind, one, [pos0[0]], [n], cos, sin, hq, hkv, dtype, gs, False)[0]
                assert not torch.equal(alt, exp), (n_tok, pos0, b)
            r0 += n
    # equal lengths: the fixed-length batched call
    n_tok, pos0 = [17, 17, 17], [33, 33, 33]
    d = varlen_data(gen, n_tok, hq, hkv, dtype, gs)
    if kind == "attn":
        assert torch.equal(attn(emu, d, pos0, n_tok, hq, dtype, True), attn(emu, d, pos0, n_tok, hq, dtype, False))
    else:
        (qa, ca), (qb, cb) = (append(emu, kind, d, pos0, n_tok, cos, sin, hq, hkv, dtype, gs, v) for v in (True, False))
        assert torch.equal(qa, qb)
        for k in ca:
            assert torch.equal(ca[k], cb[k]), k


def test_emulated_ragged_argument_checks(emu):
    """Every out-of-range host argument of the _varlen entry points, and a null position array of the _seqpos ones, is
    HQQ_E_INVALID with the entry point's name in the message."""
    buf = torch.zeros(1 << 20, dtype=torch.uint8)
    L = 64

    def rows(p0, nt, batch):
        return emu.hqq_b200_glue_rope_append_rows_varlen(*[P(buf)] * 8, ints(p0), ints(nt), 8, 2, L, R.HD, batch, F16, None)

    def rows8(p0, nt, batch):
        return emu.hqq_b200_glue_rope_append_rows_kv8_varlen(*[P(buf)] * 14, ints(p0), ints(nt), 8, 2, L, R.HD, 64, batch, F16, None)

    def att(p0, nt, batch):
        return emu.hqq_b200_glue_attn_prefill_varlen(*[P(buf)] * 4, ints(p0), ints(nt), 8, 2, L, R.HD, batch, F16, None)

    bad = [([0, 0], [-1, 2], 2), ([-1, 0], [1, 2], 2), ([60, 0], [5, 2], 2), ([0, 64], [0, 1], 2), ([0, 0], [0, 0], 2), ([0], [1], 0),
           ([0] * 257, [1] * 257, 257)]
    for fn, name in ((rows, b"rows_varlen"), (rows8, b"rows_kv8_varlen"), (att, b"attn_prefill_varlen")):
        for p0, nt, batch in bad:
            assert fn(p0, nt, batch) == E_INVALID, (name, p0, nt, batch)
            assert name in emu.hqq_b200_last_error()
    # more than 65535 rows in all
    big = 40000
    assert emu.hqq_b200_glue_attn_prefill_varlen(*[P(buf)] * 4, ints([0, 0]), ints([big, big]), 8, 2, 65536, R.HD, 2, F16, None) == E_INVALID
    assert b"65535" in emu.hqq_b200_last_error()
    # null position arrays
    assert emu.hqq_b200_glue_attn_prefill_varlen(*[P(buf)] * 4, None, ints([1]), 8, 2, L, R.HD, 1, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_rope_attn_decode_batch_seqpos(*[P(buf)] * 7, None, P(buf), 8, 2, L, R.HD, 1, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_rope_attn_decode_split_seqpos(*[P(buf)] * 7, None, P(buf), P(buf), 8, 2, L, R.HD, 1, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_rope_attn_decode_split_kv8_seqpos(*[P(buf)] * 11, None, P(buf), P(buf), 8, 2, L, R.HD, 64, 1, F16, None) == E_INVALID
    assert b"seqpos" in emu.hqq_b200_last_error()
