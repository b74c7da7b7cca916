"""The 8-bit HQQ KV cache on the H100: hqq_b200_glue_rope_attn_decode_split_kv8 at full length, and the decode harness with
kv_bits=8 (fused steps, batch, prefill, a prompt that fills the cache) against its framework-op reference.

Kernel outputs are held to the bound of tests/attn_kv8_ref.py (the split-KV bound over the dequantised cache), and the four defects
that module builds must each break it.

Harness runs are compared with the fused=False kv8 reference: logits under the split-KV tests' bars (relative L2 2e-3 fp16, 1e-2
bf16) and token rule.  Their dequantised caches get CACHE_TOL instead: the two paths' k / v rows differ by fp16 / bf16 rounding
(about 1e-3 of a row's spread), and a level is 1 / 255 of a group's range, so a few per cent of the levels sit on the other side of a
rounding boundary and move by one level -- a relative L2 of a few 1e-3 with no error in either path."""
import pytest
import torch

import attn_kv8_ref as K8
import attn_split_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
L_MAX = 131072
CACHE_TOL = {torch.float16: 1e-2, torch.bfloat16: 3e-2}


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def run_kv8(case, pos, cos, sin, hq, hkv, dtype, gs):
    lib = load()
    batch, L = case["kq"].shape[0], case["kq"].shape[2]
    c = {n: case[n].clone() for n in ("kq", "ks", "kz", "vq", "vs", "vz")}
    out = torch.zeros(batch, hq * R.HD, dtype=dtype, device=DEV)
    ws = torch.zeros(lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, batch), dtype=torch.uint8, device=DEV)
    p = torch.tensor([pos], dtype=torch.int64, device=DEV)
    check(lib.hqq_b200_glue_rope_attn_decode_split_kv8(ptr(case["q"]), ptr(case["k"]), ptr(case["v"]), ptr(cos), ptr(sin), ptr(c["kq"]), ptr(c["ks"]),
                                                       ptr(c["kz"]), ptr(c["vq"]), ptr(c["vs"]), ptr(c["vz"]), ptr(p), ptr(out), ptr(ws), hq, hkv, L, R.HD,
                                                       gs, batch, DTYPE_CODE[dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out, c, ws


POSITIONS = (0, 17, 8191, 8193, 65535, 100003, 131071)


@pytest.mark.parametrize("dtype,gs", [(torch.float16, 64), (torch.bfloat16, 128)], ids=["f16-gs64", "bf16-gs128"])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (64, 8), (8, 1)])
def test_kv8_attention_full_length_within_bound(dtype, gs, hq, hkv):
    """cache_len 131072: within the bound at every position class, the 8-bit caches as expected bit for bit (row pos quantised,
    nothing else touched), tickets back at zero, and the four defects outside the bound."""
    S = R.split_count(sms(), hkv, L_MAX)
    cos, sin = R.tables(L_MAX, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq * 10 + hkv)
    worst = 0.0
    for pos in POSITIONS:
        case = K8.make_case(gen, 1, hq, hkv, L_MAX, pos, dtype, cos, sin, gs, DEV)
        out, c, ws = run_kv8(case, pos, cos, sin, hq, hkv, dtype, gs)
        y, bound, exp = K8.reference(case, pos, cos, sin, S, dtype, gs)
        for n in exp:
            assert torch.equal(c[n], exp[n]), (pos, n)
        assert torch.count_nonzero(ws[-4 * hkv:]) == 0, pos
        ratio, ok = R.within(out, y, bound)
        assert ok, (pos, ratio)
        worst = max(worst, ratio)
        if pos >= 2:
            for name, bad in K8.defects(case, exp, pos, cos, sin, S, gs).items():
                assert not R.within(bad, y, bound)[1], (pos, name)
        del case, c, exp
    print(f"largest err / bound {worst:.3f}")


# ------------------------------------------------------------------------------------------------ harness
SHAPE = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)


def _model(fused, dtype, cache_len, batch, gs=64):
    return harness.DecodeModel(SHAPE, dtype=dtype, device=DEV, cache_len=cache_len, fused=fused, seed=3, batch=batch, kv_bits=8, kv_group_size=gs)


def _deq_caches(m, end):
    return [tuple(harness.kv8_dequantize(blk[n + "_cache"][:, :, :end], blk[n + "_scale"][:, :, :end], blk[n + "_zero"][:, :, :end]).float().clone()
                  for n in ("k", "v")) for blk in m.blocks]


def _close(got, ref, tol, what):
    for li, ((k, v), (kr, vr)) in enumerate(zip(got, ref)):
        for name, a, r in (("k", k, kr), ("v", v, vr)):
            rel = float((a - r).norm() / r.norm())
            assert rel <= tol, (what, li, name, rel)


def _agree(a, b, batch):
    """Free-running greedy tokens per sequence: the first 4 equal.  (The split-KV tests also ask 22 of 24; this random-weight model
    settles into a 1919 / 45 alternation whose logits nearly tie, and one flip -- a level on the other side of a rounding boundary
    is enough -- sends the two runs apart.  The later steps are compared teacher-forced instead.)"""
    for s in range(batch):
        x, y = [t[s] for t in a], [t[s] for t in b]
        assert x[:4] == y[:4], (s, x, y)


def _decode(fused, start, n, batch=1, cache_len=16384, gs=64, forced=None):
    """n steps from `start` over identical pre-filled caches; forced: the tokens each step after the first is fed (teacher forcing)
    instead of the previous step's output."""
    m = _model(fused, torch.float16, cache_len, batch, gs)
    m.capture()
    m.reset_state()
    g = torch.Generator(device=DEV).manual_seed(77)
    for blk in m.blocks:  # identical pre-filled caches in every model: random rows quantised
        for c in ("k", "v"):
            rows = (torch.randn(blk[c + "_cache"].shape, generator=g, device=DEV) * 0.5).half()
            lv, sc, ze = harness.kv8_quantize_rows(rows, gs)
            blk[c + "_cache"].copy_(lv); blk[c + "_scale"].copy_(sc); blk[c + "_zero"].copy_(ze)
    m.tok.copy_(torch.arange(5, 5 + batch, device=DEV))
    m.pos.fill_(start)
    toks = []
    for i in range(n):
        if forced is not None and i > 0:
            m.tok.copy_(torch.tensor(forced[i - 1], device=DEV))
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize(DEV)
    return m, toks


@pytest.mark.parametrize("gs", [64, 128])
def test_kv8_decode_across_8192_fused_steps_equal_framework_ops(gs):
    """fused=5, fused=True and a lock-step batch of 4 decode 24 tokens from 8180 over a 16384-position 8-bit cache: the same tokens
    as the fused=False kv8 reference on the first 4; fed the reference's tokens, every layer's dequantised cache within CACHE_TOL of
    the reference's and at least 22 of 24 greedy picks equal."""
    for batch in (1, 4):
        mr, tref = _decode(False, 8180, 24, batch=batch, gs=gs)
        ref_c = _deq_caches(mr, 8204)
        for fused in ((5, True) if batch == 1 else (True,)):
            m, t = _decode(fused, 8180, 24, batch=batch, gs=gs)
            assert m.attn_kernel == "split_kv8"
            _agree(t, tref, batch)
            m, tf = _decode(fused, 8180, 24, batch=batch, gs=gs, forced=tref)
            _close(_deq_caches(m, 8204), ref_c, CACHE_TOL[torch.float16], (fused, batch))
            for s in range(batch):
                assert sum(int(u[s] == v[s]) for u, v in zip(tf, tref)) >= 22, (fused, s, tf, tref)


def _prefill_then_decode(m, prompt, chunk, n=24):
    m.reset_state()
    tok = m.prefill(prompt, chunk=chunk)
    T = prompt.shape[-1]
    assert int(m.pos.item()) == T % m.cache_len and torch.equal(tok, m.tok)
    logits = m.last_logits.float().clone()
    caches = _deq_caches(m, T)
    toks = [tok.tolist()]
    for _ in range(n - 1):
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize(DEV)
    return toks, logits, caches


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("T,chunk", [(17, 64), (300, 64), (5000, 1000)])
def test_kv8_prefill_matches_framework_ops(dtype, T, chunk):
    """fused=5, fused=True and a batch of 4 against the fused=False kv8 prefill: last-position logits within 2e-3 (fp16) / 1e-2
    (bf16), dequantised caches within CACHE_TOL; in fp16 also the greedy tokens of the captured step continuing from the prefill."""
    tol = 2e-3 if dtype == torch.float16 else 1e-2
    for fused, batch in ((5, 1), (True, 1), (True, 4)):
        prompt = torch.randint(0, SHAPE.vocab, (batch, T), generator=torch.Generator(device=DEV).manual_seed(T + batch), device=DEV)
        m = _model(fused, dtype, 16384, batch)
        m.capture()
        toks, logits, caches = _prefill_then_decode(m, prompt, chunk)
        mr = _model(False, dtype, 16384, batch)
        mr.capture()
        ref, ref_logits, ref_caches = _prefill_then_decode(mr, prompt, chunk)
        _close(caches, ref_caches, CACHE_TOL[dtype], (fused, batch, "prefill"))
        rel = float((logits - ref_logits).norm() / ref_logits.norm())
        assert rel <= tol, (fused, batch, "logits", rel)
        if dtype == torch.float16:
            _agree(toks, ref, batch)


def test_kv8_prompt_filling_the_cache_wraps_like_a_step():
    for fused in (5, True):
        outs = []
        for f in (fused, False):
            m = _model(f, torch.float16, 8256, 1)
            m.capture()
            m.reset_state()
            prompt = torch.randint(0, SHAPE.vocab, (1, 8256), generator=torch.Generator(device=DEV).manual_seed(8256), device=DEV)
            tok = m.prefill(prompt, chunk=1000)
            assert int(m.pos.item()) == 0
            m.decode()
            torch.cuda.synchronize(DEV)
            assert int(m.pos.item()) == 1
            outs.append((int(tok), int(m.next_tok)))
        assert outs[0] == outs[1], (fused, outs)


@pytest.mark.parametrize("gs", [64, 128])
def test_kv8_cache_bytes_and_arguments(gs):
    m16 = harness.DecodeModel(SHAPE, dtype=torch.float16, device=DEV, cache_len=1024, fused=5, seed=3)
    m8 = _model(5, torch.float16, 1024, 1, gs)
    assert m8.kv_cache_bytes() * 256 == m16.kv_cache_bytes() * (128 + 4 * 128 // gs)
    assert m16.attn_kernel == "single" and m8.attn_kernel == "split_kv8"
    for kw in ({"kv_bits": 4}, {"kv_bits": 8, "kv_group_size": 32}, {"kv_group_size": 256}):
        with pytest.raises(ValueError):
            harness.DecodeModel(SHAPE, dtype=torch.float16, device=DEV, cache_len=64, n_layers=1, **kw)
