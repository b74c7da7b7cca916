"""Prompt prefill kernels (hqq_b200_glue_rope_append_rows, hqq_b200_glue_attn_prefill, csrc/decode_glue.cu) on the CPU kernel
emulator.

Attention outputs are held to the per-element bound of tests/attn_prefill_ref.py against causal softmax attention in float64, and
the defects that module builds from the same data (causal mask off by one, diagonal omitted, key tile 0 dropped, wrong kv head)
must each break it.  Chunk lengths and offsets sit at the 64-position tile edges and the 128-row query blocks."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
import attn_prefill_ref as R  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
E_INVALID, E_UNSUPPORTED = -1, -2
VP, I = ctypes.c_void_p, ctypes.c_int
HEADS = {1: (2, 2), 4: (8, 2), 8: (8, 1)}  # G -> (n_q, n_kv)
# (T, pos0, batch): every T in {1, 15, 16, 17, 63, 64, 65, 130} and every pos0 in {0, 1, 63, 64, 1000}, batch 1 and 3
CASES = [(1, 0, 1), (15, 1, 3), (16, 63, 1), (17, 64, 3), (63, 0, 1), (64, 1, 1), (65, 63, 1), (130, 64, 1), (1, 1000, 3), (17, 1000, 1),
         (130, 0, 1)]


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_glue_rope_append_rows.argtypes = [VP] * 8 + [I] * 8 + [VP]
    lib.hqq_b200_glue_attn_prefill.argtypes = [VP] * 4 + [I] * 8 + [VP]
    lib.hqq_b200_glue_rope_attn_decode_batch.argtypes = [VP] * 9 + [I] * 6 + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr())


def attn(emu, q, kc, vc, pos0, T, hq, hkv, dtype):
    batch, L = kc.shape[0], kc.shape[2]
    out = torch.full((batch * T, hq * R.HD), float("nan"), dtype=dtype)
    rc = emu.hqq_b200_glue_attn_prefill(P(q), P(kc), P(vc), P(out), pos0, T, hq, hkv, L, R.HD, batch, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out


def append(emu, case, cos, sin, pos0, T, hq, hkv, dtype):
    batch, L = case["kc"].shape[0], case["kc"].shape[2]
    kc, vc = case["kc"].clone(), case["vc"].clone()
    qo = torch.zeros(batch * T, hq * R.HD, dtype=dtype)
    rc = emu.hqq_b200_glue_rope_append_rows(P(case["q"]), P(case["k"]), P(case["v"]), P(cos), P(sin), P(kc), P(vc), P(qo), pos0, T, hq, hkv, L,
                                            R.HD, batch, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return qo, kc, vc


def prefill(emu, case, cos, sin, chunks, hq, hkv, dtype):
    """append + attention over consecutive chunks [(pos0, T), ...] of one prompt; rows of every chunk's output concatenated per
    sequence, and the caches."""
    batch = case["kc"].shape[0]
    tot = sum(T for _, T in chunks)
    base = chunks[0][0]
    kc, vc = case["kc"].clone(), case["vc"].clone()
    outs = torch.empty(batch, tot, hq * R.HD, dtype=dtype)
    for pos0, T in chunks:
        rows = lambda x: x.view(batch, tot, -1)[:, pos0 - base:pos0 - base + T].reshape(batch * T, -1).contiguous()
        sub = {"q": rows(case["q"]), "k": rows(case["k"]), "v": rows(case["v"]), "kc": kc, "vc": vc}
        qo, kc, vc = append(emu, sub, cos, sin, pos0, T, hq, hkv, dtype)
        outs[:, pos0 - base:pos0 - base + T] = attn(emu, qo, kc, vc, pos0, T, hq, hkv, dtype).view(batch, T, -1)
    return outs.view(batch * tot, -1), kc, vc


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("G", [1, 4, 8])
@pytest.mark.parametrize("T,pos0,B", CASES)
def test_emulated_prefill_attention_within_bound_and_defects_break_it(emu, dtype, G, T, pos0, B):
    """Every output element within the derived bound; each modelled defect of the same data outside it."""
    hq, hkv = HEADS[G]
    L = pos0 + T + 7
    gen = torch.Generator().manual_seed(100 * G + 10 * T + pos0)
    case = R.make_case(gen, B, hq, hkv, L, pos0, T, dtype, "cpu")
    out = attn(emu, case["q"], case["kc"], case["vc"], pos0, T, hq, hkv, dtype)
    y, bound = R.reference(case, pos0, T, dtype)
    ratio, ok = R.within(out, y, bound)
    assert ok, ratio
    bad = R.defects(case, pos0, T, dtype)
    assert len(bad) == (4 if hkv >= 2 else 3)
    for name, d in bad.items():
        assert not R.within(d, y, bound)[1], name


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("G", [1, 4, 8])
def test_emulated_rope_append_rows_exact_and_equal_to_decode_rows(emu, dtype, G):
    """q_out and cache rows [pos0, pos0 + T) equal attn_split_ref.rope of the inputs and v exactly, nothing else in the caches
    moves, and a row equals the row hqq_b200_glue_rope_attn_decode_batch writes at the same position from the same k and v."""
    hq, hkv = HEADS[G]
    B, L, pos0, T = 3, 300, 61, 70
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(G)
    case = R.make_append_case(gen, B, hq, hkv, L, T, dtype, "cpu")
    qo, kc, vc = append(emu, case, cos, sin, pos0, T, hq, hkv, dtype)
    qr, kr, vr = R.expected_append(case, pos0, T, cos, sin)
    assert torch.equal(qo, qr) and torch.equal(kc, kr) and torch.equal(vc, vr)
    for t in (0, 3, T - 1):
        qt, kt, vt = (case[n].view(B, T, -1)[:, t].contiguous() for n in ("q", "k", "v"))  # kept alive across the launch
        kx, vx = case["kc"].clone(), case["vc"].clone()
        ox = torch.zeros(B, hq * R.HD, dtype=dtype)
        p = torch.tensor([pos0 + t], dtype=torch.int64)
        assert emu.hqq_b200_glue_rope_attn_decode_batch(P(qt), P(kt), P(vt), P(cos), P(sin), P(kx), P(vx), P(p), P(ox), hq, hkv, L, R.HD, B, CODE[dtype],
                                                        None) == 0
        assert torch.equal(kx[:, :, pos0 + t], kc[:, :, pos0 + t]) and torch.equal(vx[:, :, pos0 + t], vc[:, :, pos0 + t]), t


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_prefill_ignores_nan_rows_past_the_chunk(emu, dtype):
    """Cache rows at or past pos0 + T filled with NaN: the output is finite and bit for bit the output without them."""
    hq, hkv, B, pos0, T = 8, 2, 1, 40, 30
    L = 200
    case = R.make_case(torch.Generator().manual_seed(3), B, hq, hkv, L, pos0, T, dtype, "cpu")
    out = attn(emu, case["q"], case["kc"], case["vc"], pos0, T, hq, hkv, dtype)
    kc, vc = case["kc"].clone(), case["vc"].clone()
    kc[:, :, pos0 + T:] = float("nan")
    vc[:, :, pos0 + T:] = float("nan")
    out2 = attn(emu, case["q"], kc, vc, pos0, T, hq, hkv, dtype)
    assert torch.isfinite(out2).all()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("G", [4, 8])
def test_emulated_prefill_chunking_batch_and_repeat_bit_identical(emu, dtype, G):
    """The same positions in one call and in two chunks split at an odd offset, a batch row and the sequence alone, and two
    identical calls give bit-identical outputs and caches."""
    hq, hkv = HEADS[G]
    B, L, pos0, T = 2, 160, 5, 90
    cos, sin = R.tables(L, dtype, "cpu")
    case = R.make_append_case(torch.Generator().manual_seed(10 + G), B, hq, hkv, L, T, dtype, "cpu")
    out, kc, vc = prefill(emu, case, cos, sin, [(pos0, T)], hq, hkv, dtype)
    out2, kc2, vc2 = prefill(emu, case, cos, sin, [(pos0, 37), (pos0 + 37, T - 37)], hq, hkv, dtype)
    assert torch.equal(out, out2) and torch.equal(kc, kc2) and torch.equal(vc, vc2)
    out3, _, _ = prefill(emu, case, cos, sin, [(pos0, T)], hq, hkv, dtype)
    assert torch.equal(out, out3)
    assert torch.isfinite(out.float()).all()
    b = 1
    one = {n: case[n].view(B, -1)[b:b + 1].reshape(T, -1).contiguous() for n in ("q", "k", "v")}
    one["kc"], one["vc"] = case["kc"][b:b + 1].clone(), case["vc"][b:b + 1].clone()
    o1, kc1, vc1 = prefill(emu, one, cos, sin, [(pos0, T)], hq, hkv, dtype)
    assert torch.equal(o1, out.view(B, T, -1)[b]) and torch.equal(kc1[0], kc[b]) and torch.equal(vc1[0], vc[b])


def test_emulated_prefill_argument_checks(emu):
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    attn_call = lambda pos0, T, hq, hkv, L, hd, B, dt=F16: emu.hqq_b200_glue_attn_prefill(P(buf), P(buf), P(buf), P(buf), pos0, T, hq, hkv, L, hd, B,
                                                                                          dt, None)
    app_call = lambda pos0, T, hq, hkv, L, hd, B, dt=F16: emu.hqq_b200_glue_rope_append_rows(P(buf), P(buf), P(buf), P(buf), P(buf), P(buf), P(buf),
                                                                                             P(buf), pos0, T, hq, hkv, L, hd, B, dt, None)
    bad = [((0, 1, 8, 1, 64, 64, 1), E_UNSUPPORTED),       # head_dim 64
           ((0, 1, 9, 2, 64, 128, 1), E_UNSUPPORTED),      # n_q % n_kv
           ((0, 1, 16, 1, 64, 128, 1), E_UNSUPPORTED),     # G = 16
           ((0, 1, 8, 1, 131073, 128, 1), E_UNSUPPORTED),  # cache_len past 131072
           ((0, 1, 8, 1, 0, 128, 1), E_UNSUPPORTED),       # cache_len 0
           ((0, 0, 8, 1, 64, 128, 1), E_INVALID),          # T = 0
           ((60, 5, 8, 1, 64, 128, 1), E_INVALID),         # pos0 + T > cache_len
           ((-1, 5, 8, 1, 64, 128, 1), E_INVALID),         # pos0 < 0
           ((0, 1, 8, 1, 64, 128, 0), E_INVALID),          # batch 0
           ((0, 1, 8, 1, 64, 128, 65536), E_INVALID)]      # batch past 65535
    for call, name in ((attn_call, b"hqq_b200_glue_attn_prefill"), (app_call, b"hqq_b200_glue_rope_append_rows")):
        for args, code in bad:
            assert call(*args) == code, (name, args)
            assert name in emu.hqq_b200_last_error()
        assert call(0, 1, 8, 1, 64, 128, 1, dt=0) == E_INVALID  # float32
    assert emu.hqq_b200_glue_attn_prefill(None, P(buf), P(buf), P(buf), 0, 1, 8, 1, 64, 128, 1, F16, None) == E_INVALID
    assert emu.hqq_b200_glue_rope_append_rows(P(buf), P(buf), None, P(buf), P(buf), P(buf), P(buf), P(buf), 0, 1, 8, 1, 64, 128, 1, F16,
                                              None) == E_INVALID
