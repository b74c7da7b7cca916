"""Split-KV decode attention on the H100 (hqq_b200_glue_rope_attn_decode_split, csrc/decode_glue.cu) and the decode harness across
the 8192-position boundary where the fused steps switch to it.

Kernel outputs are held to the per-element bound of tests/attn_split_ref.py against softmax(q k^T / sqrt(d)) v in float64, and the
three defects that module builds from the same data must each break it."""
import pytest
import torch

import attn_split_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
L_MAX = 131072


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def run_split(case, pos, cos, sin, hq, hkv, dtype, ws=None):
    lib = load()
    batch, L = case["kc"].shape[0], case["kc"].shape[2]
    kc, vc = case["kc"].clone(), case["vc"].clone()
    out = torch.zeros(batch, hq * R.HD, dtype=dtype, device=DEV)
    if ws is None:
        nbytes = lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, batch)
        assert nbytes == R.workspace_bytes(sms(), hq, hkv, batch)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    p = torch.tensor([pos], dtype=torch.int64, device=DEV)
    check(lib.hqq_b200_glue_rope_attn_decode_split(ptr(case["q"]), ptr(case["k"]), ptr(case["v"]), ptr(cos), ptr(sin), ptr(kc), ptr(vc), ptr(p),
                                                   ptr(out), ptr(ws), hq, hkv, L, R.HD, batch, DTYPE_CODE[dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out, kc, vc, ws


POSITIONS = (0, 1, 8191, 8192, 8193, 40001, 65535, 100003, 131071)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (64, 8), (8, 1)])
def test_split_attention_full_length_within_bound(dtype, hq, hkv):
    """cache_len 131072: every position class within the bound, cache rows exact, tickets back at zero, two calls bit-identical,
    and the three defects of the same data outside the bound."""
    S = R.split_count(sms(), hkv, L_MAX)
    cos, sin = R.tables(L_MAX, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq * 10 + hkv)
    worst = 0.0
    for pos in POSITIONS:
        case = R.make_case(gen, 1, hq, hkv, L_MAX, pos, dtype, cos, sin, DEV)
        out, kc, vc, ws = run_split(case, pos, cos, sin, hq, hkv, dtype)
        y, bound, kref, vref = R.reference(case, pos, cos, sin, S, dtype)
        assert torch.equal(kc, kref) and torch.equal(vc, vref), pos
        assert torch.count_nonzero(ws[-4 * hkv:]) == 0, pos
        ratio, ok = R.within(out, y, bound)
        assert ok, (pos, ratio)
        worst = max(worst, ratio)
        out2, _, _, _ = run_split(case, pos, cos, sin, hq, hkv, dtype, ws)
        assert torch.equal(out, out2), pos
        if pos >= 2:
            for name, bad in zip(("split 0 dropped", "stale row at pos", "pos - 1 omitted"), R.defects(case, pos, cos, sin, S)):
                assert not R.within(bad, y, bound)[1], (pos, name)
        del case, kc, vc, kref, vref
    print(f"largest err / bound {worst:.3f}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_split_attention_batch_rows_equal_single_sequence_calls(dtype):
    """Batch 4: every sequence gets bit for bit what it gets alone (S ignores batch)."""
    hq, hkv, B = 32, 8, 4
    cos, sin = R.tables(L_MAX, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    for pos in (8191, 70000):
        case = R.make_case(gen, B, hq, hkv, L_MAX, pos, dtype, cos, sin, DEV)
        out, kc, vc, _ = run_split(case, pos, cos, sin, hq, hkv, dtype)
        for b in range(B):
            one = {n: case[n][b:b + 1].clone() for n in ("q", "k", "v", "kc", "vc")}
            o1, kc1, vc1, _ = run_split(one, pos, cos, sin, hq, hkv, dtype)
            assert torch.equal(o1[0], out[b]) and torch.equal(kc1[0], kc[b]) and torch.equal(vc1[0], vc[b]), (pos, b)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_split_attention_cache_rows_equal_existing_kernel_at_8192(dtype):
    """cache_len 8192: the split kernel writes the cache rows the one-CTA-per-head entry point writes, bit for bit, and its output
    stays within the bound where that kernel's does."""
    lib = load()
    hq, hkv, B, L = 32, 8, 2, 8192
    S = R.split_count(sms(), hkv, L)
    cos, sin = R.tables(L, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(9)
    for pos in (0, 4097, 8191):
        case = R.make_case(gen, B, hq, hkv, L, pos, dtype, cos, sin, DEV)
        out, kc, vc, _ = run_split(case, pos, cos, sin, hq, hkv, dtype)
        kx, vx = case["kc"].clone(), case["vc"].clone()
        ox = torch.zeros_like(out)
        p = torch.tensor([pos], dtype=torch.int64, device=DEV)
        check(lib.hqq_b200_glue_rope_attn_decode_batch(ptr(case["q"]), ptr(case["k"]), ptr(case["v"]), ptr(cos), ptr(sin), ptr(kx), ptr(vx), ptr(p),
                                                       ptr(ox), hq, hkv, L, R.HD, B, DTYPE_CODE[dtype], stream_ptr(DEV)))
        torch.cuda.synchronize(DEV)
        assert torch.equal(kx, kc) and torch.equal(vx, vc), pos
        y, bound, _, _ = R.reference(case, pos, cos, sin, S, dtype)
        assert R.within(out, y, bound)[1], pos


# ------------------------------------------------------------------------------------------------ harness across 8192
SHAPE = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)


def _decode(fused, start, n, batch=1, cache_len=16384):
    m = harness.DecodeModel(SHAPE, dtype=torch.float16, device=DEV, cache_len=cache_len, fused=fused, seed=3, batch=batch)
    m.capture()
    g = torch.Generator(device=DEV).manual_seed(77)
    for blk in m.blocks:  # identical pre-filled caches in every model
        blk["k_cache"].copy_(torch.randn(blk["k_cache"].shape, generator=g, device=DEV) * 0.5)
        blk["v_cache"].copy_(torch.randn(blk["v_cache"].shape, generator=g, device=DEV) * 0.5)
    m.tok.copy_(torch.arange(5, 5 + batch, device=DEV))
    m.pos.fill_(start)
    toks = []
    for _ in range(n):
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize(DEV)
    return m, toks


@pytest.mark.parametrize("start", [8180, 0])
def test_decode_across_8192_fused_steps_equal_framework_ops(start):
    """A 2-layer model at cache_len 16384 (split-KV attention in both fused steps) decoding 24 tokens from `start`: fused=5 and
    fused=True give the same tokens; each agrees with the framework-op step on the first tokens and on all but at most two."""
    m5, t5 = _decode(5, start, 24)
    m8, t8 = _decode(True, start, 24)
    mr, tref = _decode(False, start, 24)
    assert m5.attn_kernel == "split" and m8.attn_kernel == "split"
    assert t5 == t8, (t5, t8)
    for t in (t5, t8):
        assert t[:4] == tref[:4], (t, tref)
        assert sum(int(x == y) for x, y in zip(t, tref)) >= 22, (t, tref)


def test_decode_across_8192_lock_step_batch():
    m8, t8 = _decode(True, 8180, 24, batch=4)
    mr, tref = _decode(False, 8180, 24, batch=4)
    assert m8.attn_kernel == "split"
    for s in range(4):
        a, r = [t[s] for t in t8], [t[s] for t in tref]
        assert a[:4] == r[:4], (s, a, r)
        assert sum(int(x == y) for x, y in zip(a, r)) >= 22, (s, a, r)


def test_short_cache_keeps_the_single_kernel():
    m = harness.DecodeModel(SHAPE, dtype=torch.float16, device=DEV, cache_len=32, fused=5, seed=3)
    assert m.attn_kernel == "single"
    m.capture()
    assert "attn_ws" not in m._bufs
