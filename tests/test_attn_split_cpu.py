"""Split-KV decode attention (hqq_b200_glue_rope_attn_decode_split, csrc/decode_glue.cu) on the CPU kernel emulator, and the
Llama-3.1 RoPE tables of the decode harness.

The emulator has 4 SMs, so S = max(1, min(4 / n_kv, ceil(cache_len / 16))) and each split covers many positions.  Outputs are
held to the per-element bound of tests/attn_split_ref.py against softmax(q k^T / sqrt(d)) v in float64; the three defects that
module builds from the same data must each break it."""
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
E_UNSUPPORTED = -2
VP, I = ctypes.c_void_p, ctypes.c_int


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_glue_rope_attn_decode_split.argtypes = [VP] * 10 + [I] * 6 + [VP]
    lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes.restype = ctypes.c_size_t
    lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes.argtypes = [I] * 4
    lib.hqq_b200_glue_rope_attn_decode_batch.argtypes = [VP] * 9 + [I] * 6 + [VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr())


def run_split(emu, case, pos, cos, sin, hq, hkv, dtype, ws=None):
    batch, L = case["kc"].shape[0], case["kc"].shape[2]
    kc, vc = case["kc"].clone(), case["vc"].clone()
    out = torch.zeros(batch, hq * R.HD, dtype=dtype)
    if ws is None:
        ws = torch.zeros(R.workspace_bytes(SMS, hq, hkv, batch), dtype=torch.uint8)
    p = torch.tensor([pos], dtype=torch.int64)
    rc = emu.hqq_b200_glue_rope_attn_decode_split(P(case["q"]), P(case["k"]), P(case["v"]), P(cos), P(sin), P(kc), P(vc), P(p), P(out), P(ws),
                                                 hq, hkv, L, R.HD, batch, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out, kc, vc, ws


def tickets(ws, hkv, batch):
    return ws[-4 * batch * hkv:].view(torch.int32)


def positions(L, S):
    c = R.TILE * max(1, (L // (2 * S)) // R.TILE)  # a chunk length whose S-fold fits the cache twice
    return sorted({0, 1, S * c - 1, S * c, L - 1})


CASES = [(hq, hkv, B, L) for (hq, hkv) in ((4, 1), (8, 2), (8, 1)) for B in (1, 3) for L in (100, 1000, 9000)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv,B,L", CASES)
def test_emulated_split_attention_within_bound_and_caches_exact(emu, dtype, hq, hkv, B, L):
    """Output within the derived bound at every position class (0, 1, chunk edges pos + 1 = S c and S c + 1, cache_len - 1); cache
    rows equal the rounded RoPE exactly; the tickets are back at zero; the three defects of the same data break the bound."""
    S = R.split_count(SMS, hkv, L)
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(1000 * hq + 100 * hkv + 10 * B + L)
    for pos in positions(L, S):
        case = R.make_case(gen, B, hq, hkv, L, pos, dtype, cos, sin, "cpu")
        out, kc, vc, ws = run_split(emu, case, pos, cos, sin, hq, hkv, dtype)
        y, bound, kref, vref = R.reference(case, pos, cos, sin, S, dtype)
        assert torch.equal(kc, kref) and torch.equal(vc, vref), pos
        assert torch.count_nonzero(tickets(ws, hkv, B)) == 0, pos
        ratio, ok = R.within(out, y, bound)
        assert ok, (pos, ratio)
        if pos >= 2:
            for name, bad in zip(("split 0 dropped", "stale row at pos", "pos - 1 omitted"), R.defects(case, pos, cos, sin, S)):
                assert not R.within(bad, y, bound)[1], (pos, name)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", [(4, 1), (8, 2)])
def test_emulated_split_batch_rows_equal_single_sequence_calls_and_cache_rows_equal_existing_kernel(emu, dtype, hq, hkv):
    """A sequence of a lock-step batch gets bit for bit what it gets alone (S ignores batch); below 8192 positions the cache rows
    the split kernel writes are bit-identical to those of hqq_b200_glue_rope_attn_decode_batch; one workspace serves repeated
    calls (tickets left at zero)."""
    B, L = 3, 700
    cos, sin = R.tables(L, dtype, "cpu")
    gen = torch.Generator().manual_seed(7 + hq)
    for pos in (5, 383, 699):
        case = R.make_case(gen, B, hq, hkv, L, pos, dtype, cos, sin, "cpu")
        ws = torch.zeros(R.workspace_bytes(SMS, hq, hkv, B), dtype=torch.uint8)
        out, kc, vc, _ = run_split(emu, case, pos, cos, sin, hq, hkv, dtype, ws)
        out2, _, _, _ = run_split(emu, case, pos, cos, sin, hq, hkv, dtype, ws)
        assert torch.equal(out, out2)
        for b in range(B):
            one = {n: case[n][b:b + 1].clone() for n in ("q", "k", "v", "kc", "vc")}
            o1, kc1, vc1, _ = run_split(emu, one, pos, cos, sin, hq, hkv, dtype)
            assert torch.equal(o1[0], out[b]) and torch.equal(kc1[0], kc[b]) and torch.equal(vc1[0], vc[b]), (pos, b)
        kx, vx = case["kc"].clone(), case["vc"].clone()
        ox = torch.zeros(B, hq * R.HD, dtype=dtype)
        p = torch.tensor([pos], dtype=torch.int64)
        assert emu.hqq_b200_glue_rope_attn_decode_batch(P(case["q"]), P(case["k"]), P(case["v"]), P(cos), P(sin), P(kx), P(vx), P(p), P(ox),
                                                        hq, hkv, L, R.HD, B, CODE[dtype], None) == 0
        assert torch.equal(kx, kc) and torch.equal(vx, vc), pos


def test_emulated_split_workspace_size_and_argument_checks(emu):
    for hq, hkv, B in ((4, 1, 1), (8, 2, 3), (8, 1, 2), (64, 8, 4), (32, 8, 1)):
        assert emu.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, B) == R.workspace_bytes(SMS, hq, hkv, B)
    dtype = torch.float16
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    p = torch.zeros(1, dtype=torch.int64)
    call = lambda hq, hkv, L, hd: emu.hqq_b200_glue_rope_attn_decode_split(P(buf), P(buf), P(buf), P(buf), P(buf), P(buf), P(buf), P(p), P(buf),
                                                                          P(buf), hq, hkv, L, hd, 1, CODE[dtype], None)
    for hq, hkv, L, hd in ((9, 1, 64, 128), (16, 1, 64, 128), (8, 1, 64, 64), (8, 1, 64, 256), (8, 1, 131073, 128), (8, 1, 0, 128)):
        assert call(hq, hkv, L, hd) == E_UNSUPPORTED, (hq, hkv, L, hd)
        assert b"hqq_b200_glue_rope_attn_decode_split" in emu.hqq_b200_last_error()


# ------------------------------------------------------------------------------------------------ Llama-3.1 RoPE tables
def test_llama3_rope_tables_match_transformers_and_none_is_unchanged():
    """`rope_scaling` "llama3" (factor 8, low/high frequency factors 1 and 4, original context 8192): inv_freq equals the
    transformers implementation to fp32 rounding and cos / sin to 1 ulp of T; with rope_scaling=None the tables are bit for bit
    the ones the harness has always built."""
    from hqq_b200 import harness
    mr = pytest.importorskip("transformers.modeling_rope_utils")
    from transformers import LlamaConfig
    shape = harness.LLAMA31_8B
    cfg = LlamaConfig(hidden_size=shape.hidden, num_attention_heads=shape.n_heads, num_key_value_heads=shape.n_kv_heads,
                      rope_theta=shape.rope_theta, rope_scaling=dict(shape.rope_scaling), max_position_embeddings=131072)
    inv_hf, factor = mr.ROPE_INIT_FUNCTIONS["llama3"](cfg, "cpu")
    assert factor == 1.0
    inv = harness.rope_inv_freq(shape, "cpu")
    assert inv.dtype == torch.float32
    assert torch.allclose(inv, inv_hf.float(), rtol=2.0 ** -23, atol=0.0)
    L = 20000
    t = torch.arange(L, dtype=torch.float32)
    fr = torch.outer(t, inv_hf.float())
    for dtype in (torch.float16, torch.bfloat16):
        cos, sin = harness.rope_tables(shape, L, dtype, "cpu")
        for got, ref in ((cos, torch.cat([fr.cos(), fr.cos()], -1)), (sin, torch.cat([fr.sin(), fr.sin()], -1))):
            assert torch.all((got.double() - ref.double()).abs() <= R.ulp(ref.double(), dtype)), dtype
        # rope_scaling=None: today's tables bit for bit
        plain = harness.LLAMA3_8B
        inv0 = 1.0 / (plain.rope_theta ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))
        fr0 = torch.outer(t, inv0)
        c0, s0 = harness.rope_tables(plain, L, dtype, "cpu")
        assert torch.equal(c0, torch.cat([fr0.cos(), fr0.cos()], dim=-1).to(dtype))
        assert torch.equal(s0, torch.cat([fr0.sin(), fr0.sin()], dim=-1).to(dtype))
    # the scaled and unscaled tables differ (low frequencies are stretched 8 times)
    assert not torch.equal(harness.rope_tables(shape, L, torch.float16, "cpu")[0], harness.rope_tables(harness.LLAMA3_8B, L, torch.float16, "cpu")[0])
