"""Ragged batches on the H100: the _seqpos decode attention and _varlen prefill entry points (csrc/decode_glue.cu) at the 8B, 70B
and tp-8 head shapes, and DecodeModel(ragged=True) on a 2-layer Llama-3-8B-shaped model.

Kernels: every sequence of a launch equals the existing entry point called with batch 1 on its slices, bit for bit.  Harness:
equal lengths and positions reproduce the lock-step model bit for bit; mixed prompt lengths meet the prefill tests' bars against
the fused=False ragged reference; refilling a slot leaves the other slots bit for bit alone."""
import ctypes

import pytest
import torch

import attn_split_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
HEADS = [(32, 8), (64, 8), (8, 1)]


def ints(xs):
    return (ctypes.c_int * len(xs))(*xs)


def decode(kind, seqpos, case, pos, cos, sin, hq, hkv, dtype, gs=64):
    lib, B = load(), case["q"].shape[0]
    names = ("kq", "ks", "kz", "vq", "vs", "vz") if kind == "kv8" else ("kc", "vc")
    L = case[names[0]].shape[2]
    c = {n: case[n].clone() for n in names}
    out = torch.zeros(B, hq * R.HD, dtype=dtype, device=DEV)
    p = torch.tensor(pos, dtype=torch.int64, device=DEV)
    ws = torch.zeros(lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, B), dtype=torch.uint8, device=DEV)
    sfx, code, st = "_seqpos" if seqpos else "", DTYPE_CODE[dtype], stream_ptr(DEV)
    head = [ptr(case["q"]), ptr(case["k"]), ptr(case["v"]), ptr(cos), ptr(sin)]
    if kind == "batch":
        check(getattr(lib, "hqq_b200_glue_rope_attn_decode_batch" + sfx)(*head, ptr(c["kc"]), ptr(c["vc"]), ptr(p), ptr(out), hq, hkv, L, R.HD, B, code, st))
    elif kind == "split":
        check(getattr(lib, "hqq_b200_glue_rope_attn_decode_split" + sfx)(*head, ptr(c["kc"]), ptr(c["vc"]), ptr(p), ptr(out), ptr(ws), hq, hkv, L, R.HD, B,
                                                                         code, st))
    else:
        check(getattr(lib, "hqq_b200_glue_rope_attn_decode_split_kv8" + sfx)(*head, *[ptr(c[n]) for n in names], ptr(p), ptr(out), ptr(ws), hq, hkv, L,
                                                                             R.HD, gs, B, code, st))
    torch.cuda.synchronize(DEV)
    assert torch.count_nonzero(ws[-4 * B * hkv:]) == 0
    return out, c


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
@pytest.mark.parametrize("kind", ["batch", "split", "kv8"])
def test_seqpos_decode_equals_batch1_per_sequence(kind, hq, hkv, dtype):
    """Positions up to 8191 (batch kernel) and 131071 (split, kv8) mixed in one launch: each sequence's output and caches equal the
    lock-step entry point's at batch 1, bit for bit."""
    L = 8192 if kind == "batch" else 131072
    pos = [L - 1, 0, 4097, 17] if kind == "batch" else [L - 1, 0, 70001, 8192]
    B = len(pos)
    cos, sin = R.tables(L, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq + hkv)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV).to(dtype)
    case = {"q": rn(B, hq * R.HD), "k": rn(B, hkv * R.HD), "v": rn(B, hkv * R.HD)}
    if kind == "kv8":
        for n in ("kq", "vq"):
            case[n] = torch.randint(0, 256, (B, hkv, L, R.HD), generator=gen, device=DEV, dtype=torch.uint8)
        for n in ("ks", "vs"):
            case[n] = (torch.rand(B, hkv, L, 2, generator=gen, device=DEV) * 0.02 + 0.005).to(dtype)
        for n in ("kz", "vz"):
            case[n] = (torch.rand(B, hkv, L, 2, generator=gen, device=DEV) * 255).to(dtype)
    else:
        case["kc"], case["vc"] = rn(B, hkv, L, R.HD), rn(B, hkv, L, R.HD)
    out, c = decode(kind, True, case, pos, cos, sin, hq, hkv, dtype)
    for b in range(B):
        one = {n: t[b:b + 1].clone() for n, t in case.items()}
        o1, c1 = decode(kind, False, one, [pos[b]], cos, sin, hq, hkv, dtype)
        assert torch.equal(out[b:b + 1], o1), b
        for n in c1:
            assert torch.equal(c[n][b:b + 1], c1[n]), (b, n)
        del one, c1


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
def test_varlen_prefill_equals_batch1_per_slot(hq, hkv, dtype):
    """n_tok [1000, 0, 333, 1] at pos0 [0, 5, 131072 - 333, 131071]: rows kernel and attention of every slot equal the fixed-length
    entry points at batch 1, bit for bit; the empty slot's caches are untouched."""
    lib, code, st = load(), DTYPE_CODE[dtype], stream_ptr(DEV)
    L, n_tok, pos0 = 131072, [1000, 0, 333, 1], [0, 5, 131072 - 333, 131071]
    B, M = len(n_tok), sum(n_tok)
    cos, sin = R.tables(L, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq * 3 + hkv)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV).to(dtype)
    q, k, v, kc, vc = rn(M, hq * R.HD), rn(M, hkv * R.HD), rn(M, hkv * R.HD), rn(B, hkv, L, R.HD), rn(B, hkv, L, R.HD)
    kc0, vc0 = kc.clone(), vc.clone()
    qo, out = torch.zeros_like(q), torch.zeros_like(q)
    check(lib.hqq_b200_glue_rope_append_rows_varlen(ptr(q), ptr(k), ptr(v), ptr(cos), ptr(sin), ptr(kc), ptr(vc), ptr(qo), ints(pos0), ints(n_tok), hq,
                                                    hkv, L, R.HD, B, code, st))
    check(lib.hqq_b200_glue_attn_prefill_varlen(ptr(qo), ptr(kc), ptr(vc), ptr(out), ints(pos0), ints(n_tok), hq, hkv, L, R.HD, B, code, st))
    torch.cuda.synchronize(DEV)
    r0 = 0
    for b in range(B):
        n = n_tok[b]
        if n == 0:
            assert torch.equal(kc[b], kc0[b]) and torch.equal(vc[b], vc0[b])
            continue
        k1, v1 = kc0[b:b + 1].clone(), vc0[b:b + 1].clone()
        q1, o1 = torch.zeros(n, hq * R.HD, dtype=dtype, device=DEV), torch.zeros(n, hq * R.HD, dtype=dtype, device=DEV)
        check(lib.hqq_b200_glue_rope_append_rows(ptr(q[r0:r0 + n]), ptr(k[r0:r0 + n]), ptr(v[r0:r0 + n]), ptr(cos), ptr(sin), ptr(k1), ptr(v1), ptr(q1),
                                                 pos0[b], n, hq, hkv, L, R.HD, 1, code, st))
        check(lib.hqq_b200_glue_attn_prefill(ptr(q1), ptr(k1), ptr(v1), ptr(o1), pos0[b], n, hq, hkv, L, R.HD, 1, code, st))
        torch.cuda.synchronize(DEV)
        assert torch.equal(qo[r0:r0 + n], q1) and torch.equal(out[r0:r0 + n], o1), b
        assert torch.equal(kc[b:b + 1], k1) and torch.equal(vc[b:b + 1], v1), b
        r0 += n


# ------------------------------------------------------------------------------------------------ DecodeModel(ragged=True)
SHAPE = harness.LLAMA3_8B
# the model the prefill tests' bars were set on (tests/test_attn_prefill_gpu.py, tests/test_kv8_gpu.py)
SMALL = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
CACHE_TOL_KV8 = {torch.float16: 1e-2, torch.bfloat16: 3e-2}  # tests/test_kv8_gpu.py
_MODELS = {}


def _model(dtype, ragged, fused=True, kv_bits=16, cache_len=2048, shape=SHAPE, **kw):
    key = (dtype, ragged, fused, kv_bits, cache_len, shape.hidden, tuple(sorted(kw.items())))
    if key not in _MODELS:
        m = harness.DecodeModel(shape, n_layers=2, dtype=dtype, device=DEV, cache_len=cache_len, fused=fused, seed=11, batch=4, ragged=ragged,
                                kv_bits=kv_bits, **kw)
        m.capture()
        _MODELS[key] = m
    return _MODELS[key]


def _caches(m, b, end):
    out = []
    for blk in m.blocks:
        if m.kv_bits == 8:
            out += [harness.kv8_dequantize(blk[n + "_cache"][b, :, :end], blk[n + "_scale"][b, :, :end], blk[n + "_zero"][b, :, :end]).float()
                    for n in ("k", "v")]
        else:
            out += [blk[n][b, :, :end].float().clone() for n in ("k_cache", "v_cache")]
    return out


def _steps(m, n, forced=None):
    """n captured steps: tokens and logits per step (forced: feed these tokens instead of the model's own)."""
    toks, logits = [], []
    for i in range(n):
        if forced is not None:
            m.tok.copy_(forced[i])
        m.graph.replay()
        toks.append(m.next_tok.clone())
        if m.fused:
            logits.append(m._bufs["logits"].clone())
        m.tok.copy_(m.next_tok)
    torch.cuda.synchronize(DEV)
    return toks, logits


def _prompts(lengths, seed, vocab=SHAPE.vocab):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, vocab, (n,), generator=g, device=DEV) for n in lengths]


@pytest.mark.parametrize("kv_bits", [16, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_ragged_equal_lengths_equal_lock_step(dtype, kv_bits):
    """Equal prompt lengths: prefill tokens, last_logits, caches and 16 captured steps' tokens and logits of ragged=True equal
    ragged=False bit for bit."""
    prompt = torch.randint(0, SHAPE.vocab, (4, 300), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    res = []
    for ragged in (False, True):
        m = _model(dtype, ragged, kv_bits=kv_bits)
        m.reset_state()
        tok = m.prefill(prompt, chunk=128)
        assert m.pos.tolist() == ([300] * 4 if ragged else [300])
        caches = [_caches(m, b, 300) for b in range(4)]
        res.append((tok, m.last_logits.clone(), caches, _steps(m, 16)))
    (ta, la, ca, (sa, ga)), (tb, lb, cb, (sb, gb)) = res
    assert torch.equal(ta, tb) and torch.equal(la, lb)
    for x, y in zip(ca, cb):
        assert all(torch.equal(u, w) for u, w in zip(x, y))
    assert all(torch.equal(u, w) for u, w in zip(sa, sb)) and all(torch.equal(u, w) for u, w in zip(ga, gb))


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("kv_bits,cache_len", [(16, 2048), (16, 16384), (8, 2048)], ids=["single", "split", "kv8"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_ragged_mixed_lengths_match_reference(dtype, kv_bits, cache_len):
    """Prompts of 1, 37, 300 and 1000 tokens in one packed prefill (chunk 256) and 8 teacher-forced captured steps against the
    fused=False ragged reference, on the model the prefill tests' bars were set on: logits within relative L2 2e-3 (fp16) / 1e-2
    (bf16), caches within the same bar (kv8: the kv8 tests' cache bar), and the prefill's picks an argmax of the reference logits
    up to the two paths' difference.
    kv8 fp16 gets 5e-3 on the logits: the packed rows go through the linears at M = 1338, where the 1-token slot's k row is
    rounded differently from the reference's M = 1 product, and one 8-bit level on the other side of a rounding boundary moves a
    cache row by a whole step (measured 4.8e-3 on that slot, 1.4e-3 or less on the others)."""
    tol = 2e-3 if dtype == torch.float16 else 1e-2
    if kv_bits == 8 and dtype == torch.float16:
        tol = 5e-3
    ctol = tol if kv_bits == 16 else CACHE_TOL_KV8[dtype]
    lengths = [1, 37, 300, 1000]
    prompts = _prompts(lengths, 7, SMALL.vocab)
    m = _model(dtype, True, kv_bits=kv_bits, cache_len=cache_len, shape=SMALL)
    r = _model(dtype, True, fused=False, kv_bits=kv_bits, cache_len=cache_len, shape=SMALL)
    for x in (m, r):
        x.reset_state()
    tok, rtok = m.prefill(prompts, chunk=256), r.prefill(prompts, chunk=256)
    assert m.pos.tolist() == lengths == r.pos.tolist()
    assert _rel(m.last_logits, r.last_logits) <= tol
    gap = 2 * float((m.last_logits.float() - r.last_logits.float()).abs().max())
    picked = r.last_logits.float().gather(1, tok.view(-1, 1)).squeeze(1)
    assert torch.all(picked >= r.last_logits.float().max(-1).values - gap), (tok, rtok)
    for b, n in enumerate(lengths):
        for u, w in zip(_caches(m, b, n), _caches(r, b, n)):
            assert _rel(u, w) <= ctol, (b, "prefill", _rel(u, w))
    m.tok.copy_(rtok)
    forced, _ = _steps(r, 8)
    _steps(m, 8, forced=[rtok] + forced[:-1])
    for b, n in enumerate(lengths):
        for u, w in zip(_caches(m, b, n + 8), _caches(r, b, n + 8)):
            assert _rel(u, w) <= ctol, (b, "teacher-forced", _rel(u, w))


@pytest.mark.parametrize("kv_bits", [16, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_ragged_slot_refill(dtype, kv_bits):
    """Decode 6 steps, refill slot 2 over its dirty cache, decode 8 more: slots 0, 1, 3 keep the tokens and logits of a run without
    the refill bit for bit, and slot 2's equal the same refill onto a zeroed cache."""
    m = _model(dtype, True, kv_bits=kv_bits)
    prompts, refill = _prompts([5, 40, 17, 100], 3), _prompts([23], 4)[0]
    runs = {}
    for mode in ("none", "refill", "zeroed"):
        m.reset_state()
        m.prefill(prompts, chunk=64)
        t1, g1 = _steps(m, 6)
        if mode != "none":
            if mode == "zeroed":
                for blk in m.blocks:
                    for name in ("k_cache", "v_cache", "k_scale", "k_zero", "v_scale", "v_zero"):
                        if name in blk:
                            blk[name][2].zero_()
            tok = m.prefill([None, None, refill, None], chunk=16)
            assert m.pos.tolist() == [5 + 6, 40 + 6, 23, 100 + 6]
            assert int(tok[2]) == int(m.tok[2])
        t2, g2 = _steps(m, 8)
        runs[mode] = (torch.stack(t1 + t2), torch.stack(g1 + g2))
    (tn, gn), (tr, gr), (tz, gz) = runs["none"], runs["refill"], runs["zeroed"]
    keep = [0, 1, 3]
    assert torch.equal(tn[:, keep], tr[:, keep]) and torch.equal(gn[:, keep], gr[:, keep])
    assert torch.equal(tr[6:, 2], tz[6:, 2]) and torch.equal(gr[6:, 2], gz[6:, 2])


def test_ragged_sampling_top_k_1_is_greedy():
    """do_sample with top_k=1 reproduces the greedy ragged stream bit for bit, prefill and refill included."""
    prompts, refill = _prompts([1, 37, 300, 64], 5), _prompts([9], 6)[0]
    out = []
    for kw in ({}, {"do_sample": True, "top_k": 1, "temperature": 0.7}):
        m = _model(torch.float16, True, **kw)
        m.reset_state()
        t0 = m.prefill(prompts, chunk=128)
        a, _ = _steps(m, 8)
        t1 = m.prefill([refill, None, None, None])
        b, _ = _steps(m, 8)
        out.append((t0, t1, torch.stack(a + b)))
    assert all(torch.equal(x, y) for x, y in zip(out[0], out[1]))


def test_ragged_prefill_rejects_bad_prompts():
    m = _model(torch.float16, True)
    p = _prompts([4], 1)[0]
    for bad, kw in (([p, p, p], {}), ([None] * 4, {}), ([p, None, None, torch.zeros(0, dtype=torch.long, device=DEV)], {}),
                    ([p, None, None, None], {"start": 2046}), ([p, None, None, None], {"start": [0, 0, 0]}),
                    ([p, None, None, None], {"start": -1}), (p, {})):
        with pytest.raises(ValueError):
            m.prefill(bad, **kw)
