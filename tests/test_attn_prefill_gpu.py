"""Prompt prefill on the H100: the kernels (hqq_b200_glue_rope_append_rows, hqq_b200_glue_attn_prefill, csrc/decode_glue.cu) and
DecodeModel.prefill.

Kernel outputs are held to the per-element bound of tests/attn_prefill_ref.py against causal softmax attention in float64 at the
8B (32/8), 70B (64/8) and tp-8 (8/1) head shapes with caches of 131072 positions, and the modelled defects must each break it.
The harness runs a 2-layer model through prefill and greedy decode against the framework-op prefill and against the prompt fed
token by token through the captured decode step."""
import os
import subprocess
import sys

import pytest
import torch

import attn_prefill_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
L_MAX = 131072


def attn(q, kc, vc, pos0, T, hq, hkv, dtype):
    batch, L = kc.shape[0], kc.shape[2]
    out = torch.full((batch * T, hq * R.HD), float("nan"), dtype=dtype, device=DEV)
    check(load().hqq_b200_glue_attn_prefill(ptr(q), ptr(kc), ptr(vc), ptr(out), pos0, T, hq, hkv, L, R.HD, batch, DTYPE_CODE[dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out


def append(case, cos, sin, pos0, T, hq, hkv, dtype, kc=None, vc=None):
    batch, L = case["kc"].shape[0], case["kc"].shape[2]
    kc = case["kc"].clone() if kc is None else kc
    vc = case["vc"].clone() if vc is None else vc
    qo = torch.zeros(batch * T, hq * R.HD, dtype=dtype, device=DEV)
    check(load().hqq_b200_glue_rope_append_rows(ptr(case["q"]), ptr(case["k"]), ptr(case["v"]), ptr(cos), ptr(sin), ptr(kc), ptr(vc), ptr(qo), pos0, T,
                                                hq, hkv, L, R.HD, batch, DTYPE_CODE[dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return qo, kc, vc


HEADS = [(32, 8), (64, 8), (8, 1)]
# (pos0, T): a first chunk, query blocks across a tile edge mid-cache, and chunks that end at the last cache row
SPANS = [(0, 1000), (8191, 130), (65536 - 17, 300), (L_MAX - 333, 333), (L_MAX - 1, 1)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
def test_prefill_attention_within_bound_and_defects_break_it(dtype, hq, hkv):
    worst = 0.0
    for i, (pos0, T) in enumerate(SPANS):
        gen = torch.Generator(device=DEV).manual_seed(hq + 7 * i)
        case = R.make_case(gen, 1, hq, hkv, L_MAX, pos0, T, dtype, DEV)
        out = attn(case["q"], case["kc"], case["vc"], pos0, T, hq, hkv, dtype)
        y, bound = R.reference(case, pos0, T, dtype)
        ratio, ok = R.within(out, y, bound)
        assert ok, (pos0, T, ratio)
        worst = max(worst, ratio)
        for name, bad in R.defects(case, pos0, T, dtype).items():
            assert not R.within(bad, y, bound)[1], (pos0, T, name)
        assert torch.equal(out, attn(case["q"], case["kc"], case["vc"], pos0, T, hq, hkv, dtype)), (pos0, T)
        del case, y, bound
    print(f"largest err / bound {worst:.3f}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
def test_prefill_chunking_and_batch_bit_identical(dtype, hq, hkv):
    """Append + attention over 1001 positions ending at the last cache row in one call, and in two chunks split at an odd
    offset: same outputs and caches bit for bit; a sequence of a batch of 3 gets what it gets alone."""
    B, T = 3, 1001
    pos0 = L_MAX - T
    cos, sin = R.tables(L_MAX, dtype, DEV)
    case = R.make_append_case(torch.Generator(device=DEV).manual_seed(hq), B, hq, hkv, L_MAX, T, dtype, DEV)
    rows = lambda x, a, n: x.view(B, T, -1)[:, a:a + n].reshape(B * n, -1).contiguous()

    def run(c, chunks):
        batch = c["kc"].shape[0]
        kc, vc = c["kc"].clone(), c["vc"].clone()
        outs = []
        for a, n in chunks:
            sub = {k: (rows(c[k], a, n) if batch == B else c[k].view(T, -1)[a:a + n].contiguous()) for k in ("q", "k", "v")}
            sub["kc"] = kc
            qo, _, _ = append(sub, cos, sin, pos0 + a, n, hq, hkv, dtype, kc, vc)
            outs.append(attn(qo, kc, vc, pos0 + a, n, hq, hkv, dtype).view(batch, n, -1))
        return torch.cat(outs, 1), kc, vc

    out, kc, vc = run(case, [(0, T)])
    out2, kc2, vc2 = run(case, [(0, 333), (333, T - 333)])
    assert torch.equal(out, out2) and torch.equal(kc, kc2) and torch.equal(vc, vc2)
    assert torch.isfinite(out.float()).all()
    b = 2
    one = {k: case[k].view(B, -1)[b].view(T, -1).contiguous() for k in ("q", "k", "v")}
    one["kc"], one["vc"] = case["kc"][b:b + 1].clone(), case["vc"][b:b + 1].clone()
    o1, kc1, vc1 = run(one, [(0, T)])
    assert torch.equal(o1[0], out[b]) and torch.equal(kc1[0], kc[b]) and torch.equal(vc1[0], vc[b])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
def test_appended_rows_equal_the_decode_kernels_rows(dtype, hq, hkv):
    """Rows written by hqq_b200_glue_rope_append_rows equal attn_split_ref.rope(k) and v, and the rows the one-CTA-per-head decode
    kernel (cache_len 8192) and the split-KV decode kernel (cache_len 131072) write at the same position from the same k and v."""
    lib = load()
    B, T = 2, 64
    for L, pos0 in ((8192, 8192 - T), (L_MAX, 100000)):
        cos, sin = R.tables(L, dtype, DEV)
        case = R.make_append_case(torch.Generator(device=DEV).manual_seed(L + hq), B, hq, hkv, L, T, dtype, DEV)
        qo, kc, vc = append(case, cos, sin, pos0, T, hq, hkv, dtype)
        qr, kr, vr = R.expected_append(case, pos0, T, cos, sin)
        assert torch.equal(qo, qr) and torch.equal(kc, kr) and torch.equal(vc, vr), L
        ws = None
        if L > 8192:
            ws = torch.zeros(lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, B), dtype=torch.uint8, device=DEV)
        for t in (0, 31, T - 1):
            qt, kt, vt = (case[n].view(B, T, -1)[:, t].contiguous() for n in ("q", "k", "v"))  # kept alive across the launch
            kx, vx = case["kc"].clone(), case["vc"].clone()
            ox = torch.zeros(B, hq * R.HD, dtype=dtype, device=DEV)
            p = torch.tensor([pos0 + t], dtype=torch.int64, device=DEV)
            args = (ptr(qt), ptr(kt), ptr(vt), ptr(cos), ptr(sin), ptr(kx), ptr(vx), ptr(p), ptr(ox))
            if ws is None:
                check(lib.hqq_b200_glue_rope_attn_decode_batch(*args, hq, hkv, L, R.HD, B, DTYPE_CODE[dtype], stream_ptr(DEV)))
            else:
                check(lib.hqq_b200_glue_rope_attn_decode_split(*args, ptr(ws), hq, hkv, L, R.HD, B, DTYPE_CODE[dtype], stream_ptr(DEV)))
            torch.cuda.synchronize(DEV)
            assert torch.equal(kx[:, :, pos0 + t], kc[:, :, pos0 + t]) and torch.equal(vx[:, :, pos0 + t], vc[:, :, pos0 + t]), (L, t)
        del case, kc, vc, kr, vr


# ------------------------------------------------------------------------------------------------ DecodeModel.prefill
SHAPE = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
_MODELS = {}


def _model(fused, dtype, cache_len, batch):
    key = (fused, dtype, cache_len, batch)
    if key not in _MODELS:
        m = harness.DecodeModel(SHAPE, dtype=dtype, device=DEV, cache_len=cache_len, fused=fused, seed=3, batch=batch)
        m.capture()
        _MODELS[key] = m
    return _MODELS[key]


def _prefill_then_decode(m, prompt, chunk, n=24, split_at=None):
    """[the prefill's token] + n - 1 greedy tokens (per sequence), the prefill's last-position logits, each layer's caches over the
    prompt right after the prefill, and each layer's caches over prompt + decoded positions at the end."""
    T = prompt.shape[-1]
    m.reset_state()
    if split_at is None:
        tok = m.prefill(prompt, chunk=chunk)
    else:
        m.prefill(prompt[..., :split_at], chunk=chunk)
        tok = m.prefill(prompt[..., split_at:], start=split_at, chunk=chunk)
    assert int(m.pos.item()) == T and torch.equal(tok, m.tok)
    logits = m.last_logits.float().clone()
    assert torch.equal(tok, torch.argmax(logits, dim=-1)), (tok, logits.max(-1))  # the first index of the maximum
    caches = _caches(m, T)
    toks = [tok.tolist()]
    for _ in range(n - 1):
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize(DEV)
    return toks, logits, caches, _caches(m, T + n - 1)


def _caches(m, end):
    return [(blk["k_cache"][:, :, :end].float().clone(), blk["v_cache"][:, :, :end].float().clone()) for blk in m.blocks]


def _teacher_forced(m, prompt, chunk, forced):
    """prefill, then the captured step fed the given tokens (not its own): each layer's caches over prompt + fed positions."""
    T = prompt.shape[-1]
    m.reset_state()
    m.prefill(prompt, chunk=chunk)
    for t in forced:
        m.tok.copy_(torch.tensor(t, device=DEV))
        m.graph.replay()
    torch.cuda.synchronize(DEV)
    return _caches(m, T + len(forced))


def _token_by_token(m, prompt, n=24):
    m.reset_state()
    for i in range(prompt.shape[1]):
        m.tok.copy_(prompt[:, i])
        m.graph.replay()
    m.tok.copy_(m.next_tok)
    toks = [m.tok.tolist()]
    for _ in range(n - 1):
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize(DEV)
    return toks


def _agree(a, b, batch):
    """The split-KV tests' rule per sequence: the first 4 tokens equal and at least 22 of 24."""
    for s in range(batch):
        x, y = [t[s] for t in a], [t[s] for t in b]
        assert x[:4] == y[:4], (s, x, y)
        assert sum(int(u == v) for u, v in zip(x, y)) >= 22, (s, x, y)


def _close(got, ref, tol, what):
    for li, ((k, v), (kr, vr)) in enumerate(zip(got, ref)):
        for name, a, r in (("k", k, kr), ("v", v, vr)):
            rel = float((a - r).norm() / r.norm())
            assert rel <= tol, (what, li, name, rel)


PROMPTS = [(1, 1), (17, 17), (17, 64), (300, 300), (300, 64), (300, 1000), (5000, 5000), (5000, 1000), (5000, 64)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("cache_len", [4096, 16384])
@pytest.mark.parametrize("T,chunk", PROMPTS)
def test_harness_prefill_matches_framework_ops_and_token_by_token(dtype, cache_len, T, chunk):
    """fused=5, fused=True and a batch of 4, against the framework-op prefill + step(), both dtypes:
      - every layer's caches after the prefill and the last-position logits within the forward-parity bar of DESIGN 4;
      - the returned token is the argmax of the prefill's logits, and an argmax of the framework-op logits up to their difference;
      - teacher-forced hand-off: the captured step fed the framework run's 23 tokens leaves every layer's caches over prompt + 23
        positions within the bar of the framework run's.
    In fp16 also the free-running greedy tokens (first 4 equal, at least 22 of 24) against the framework-op prefill + step() and
    against the prompt fed token by token through the same captured step.  bf16 has no free-running token rule: this
    random-weight model's bf16 greedy tokens part after a few steps between any two paths, two framework-op runs included."""
    if T + 24 > cache_len:
        pytest.skip("prompt + 24 tokens do not fit the cache")
    tol = 2e-3 if dtype == torch.float16 else 1e-2
    for fused, batch in ((5, 1), (True, 1), (True, 4)):
        prompt = torch.randint(0, SHAPE.vocab, (batch, T), generator=torch.Generator(device=DEV).manual_seed(T + batch), device=DEV)
        m = _model(fused, dtype, cache_len, batch)
        assert m.attn_kernel == ("split" if cache_len > harness.SINGLE_ATTN_MAX_LEN else "single")
        toks, logits, caches, _ = _prefill_then_decode(m, prompt, chunk)
        ref, ref_logits, ref_caches, ref_after = _prefill_then_decode(_model(False, dtype, cache_len, batch), prompt, chunk)
        _close(caches, ref_caches, tol, (fused, batch, "prefill"))
        rel = float((logits - ref_logits).norm() / ref_logits.norm())
        assert rel <= tol, (fused, batch, "logits", rel)
        gap = 2 * float((logits - ref_logits).abs().max())
        picked = ref_logits.gather(1, torch.tensor(toks[0], device=DEV).view(-1, 1)).squeeze(1)
        assert torch.all(picked >= ref_logits.max(-1).values - gap), (fused, batch, toks[0])
        _close(_teacher_forced(m, prompt, chunk, ref[:-1]), ref_after, tol, (fused, batch, "teacher-forced decode"))
        if dtype == torch.float16:
            _agree(toks, ref, batch)
            _agree(toks, _token_by_token(m, prompt), batch)


@pytest.mark.parametrize("cache_len", [64, 8256])
def test_harness_prompt_filling_the_cache_wraps_like_a_step(cache_len):
    """A prompt over every cache position: pos wraps to 0 as a step at the last position does, and the captured step (single or
    split attention) then runs at position 0 as it does after a step at the last position -- against the framework-op model."""
    for fused in (5, True):
        m, mr = _model(fused, torch.float16, cache_len, 1), _model(False, torch.float16, cache_len, 1)
        prompt = torch.randint(0, SHAPE.vocab, (1, cache_len), generator=torch.Generator(device=DEV).manual_seed(cache_len), device=DEV)
        outs = []
        for x in (m, mr):
            x.reset_state()
            tok = x.prefill(prompt, chunk=1000)
            assert int(x.pos.item()) == 0
            x.decode()
            torch.cuda.synchronize(DEV)
            assert int(x.pos.item()) == 1
            outs.append((int(tok), int(x.next_tok), x.blocks[-1]["k_cache"][0, :, 0].float().clone()))
        assert outs[0][:2] == outs[1][:2], (fused, outs[0][:2], outs[1][:2])
        assert float((outs[0][2] - outs[1][2]).norm() / outs[1][2].norm()) <= 2e-3


def test_harness_prefill_batch_with_a_vocabulary_not_a_multiple_of_8():
    """batch 3, vocabulary 2050: each row's greedy pick is the first index of its maximum, as torch.argmax has it, and the
    framework-op prefill picks the same tokens."""
    shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2050)
    prompt = torch.randint(0, shape.vocab, (3, 40), generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    toks = []
    for fused in (True, False):
        m = harness.DecodeModel(shape, dtype=torch.float16, device=DEV, cache_len=128, fused=fused, seed=4, batch=3)
        tok = m.prefill(prompt, chunk=16)
        torch.cuda.synchronize(DEV)
        assert torch.equal(tok, torch.argmax(m.last_logits, dim=-1))
        toks.append(tok.tolist())
    assert toks[0] == toks[1], toks


@pytest.mark.parametrize("fused", [5, True])
def test_harness_prefill_in_two_calls(fused):
    """prefill(tokens[:a]) then prefill(tokens[a:], start=a): pos and tok as specified, tokens as the framework-op prefill."""
    T, a = 700, 301
    prompt = torch.randint(0, SHAPE.vocab, (1, T), generator=torch.Generator(device=DEV).manual_seed(11), device=DEV)
    m = _model(fused, torch.float16, 16384, 1)
    toks = _prefill_then_decode(m, prompt[0], 256, split_at=a)[0]
    ref = _prefill_then_decode(_model(False, torch.float16, 16384, 1), prompt, 256)[0]
    _agree(toks, ref, 1)


def test_harness_prefill_rejects_bad_prompts():
    m = _model(5, torch.float16, 4096, 1)
    with pytest.raises(ValueError):
        m.prefill(torch.zeros(1, 4097, dtype=torch.long, device=DEV))
    with pytest.raises(ValueError):
        m.prefill(torch.zeros(2, 10, dtype=torch.long, device=DEV))
    with pytest.raises(ValueError):
        m.prefill(torch.zeros(1, 10, dtype=torch.long, device=DEV), start=4090)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tensor_parallel_prefill_matches_one_gpu():
    """tp = 2 prefill + decode against the one-GPU model of the same weights (both built with shard_from_full)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", "29547", os.path.join(root, "tools", "tp_prefill_check.py")], capture_output=True, text=True, timeout=600)
    assert "PREFILL-TP AGREE" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
