"""The 4-bit HQQ KV cache on the H100: hqq_b200_glue_rope_attn_decode_split_kv4 at full length, and the decode harness with
kv_bits=4 against itself (paged / unpaged, ragged / lock-step, score / prefill, sampled / greedy, speculative) bit for bit and
against its fused=False framework-op reference.

Kernel outputs are held to the bound of tests/attn_kv4_ref.py (the split-KV bound over the dequantised cache), and the defects that
module builds must each break it.

Against the reference, the last-position logits of a prefill meet the 8-bit cache's bars (relative L2 2e-3 fp16, 1e-2 bf16) widened
by sqrt(255 / 15) for the coarser levels (FLIP_SCALE below).  The
caches are compared by level: the two paths' k / v rows differ by fp16 / bf16 rounding, so a level that sits on a rounding boundary
can move by one; every differing level must be off by exactly one, and the share that differ is printed.  (The dequantised caches are
not held to one level of their group element by element: the same rounding also moves a group's min / max, hence its scale and zero,
so an element can differ by more than one level of either path's scale without any level being off by more than one.)"""
import gc

import pytest
import torch

import attn_kv4_ref as K4
import attn_split_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
L_MAX = 131072
PG = harness.KV_PAGE
SHAPE = harness.LlamaShape(hidden=4096, inter=14336, n_layers=2, n_heads=32, n_kv_heads=8, vocab=128256)
NAMES = ("kq", "ks", "kz", "vq", "vs", "vz")


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def run_kv4(case, pos, cos, sin, hq, hkv, dtype, gs):
    lib = load()
    batch, L = case["kq"].shape[0], case["kq"].shape[2]
    c = {n: case[n].clone() for n in NAMES}
    out = torch.zeros(batch, hq * R.HD, dtype=dtype, device=DEV)
    ws = torch.zeros(lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, batch), dtype=torch.uint8, device=DEV)
    p = torch.tensor([pos], dtype=torch.int64, device=DEV)
    check(lib.hqq_b200_glue_rope_attn_decode_split_kv4(ptr(case["q"]), ptr(case["k"]), ptr(case["v"]), ptr(cos), ptr(sin), *[ptr(c[n]) for n in NAMES],
                                                       ptr(p), ptr(out), ptr(ws), hq, hkv, L, R.HD, gs, batch, DTYPE_CODE[dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out, c, ws


POSITIONS = (0, 17, 8193, 65535, 100003, 131071)


@pytest.mark.parametrize("gs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (64, 8), (8, 1)])
def test_kv4_attention_full_length_within_bound(dtype, gs, hq, hkv):
    """cache_len 131072 at the 8B, 70B and tp-8 head shapes: within the bound at every position class, the 4-bit caches as expected
    bit for bit (row pos quantised and packed, nothing else touched), tickets back at zero, and the defects outside the bound."""
    S = R.split_count(sms(), hkv, L_MAX)
    cos, sin = R.tables(L_MAX, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq * 10 + hkv + gs)
    worst = 0.0
    for pos in POSITIONS:
        case = K4.make_case(gen, 1, hq, hkv, L_MAX, pos, dtype, cos, sin, gs, DEV)
        out, c, ws = run_kv4(case, pos, cos, sin, hq, hkv, dtype, gs)
        y, bound, exp = K4.reference(case, pos, cos, sin, S, dtype, gs)
        for n in exp:
            assert torch.equal(c[n], exp[n]), (pos, n)
        assert torch.count_nonzero(ws[-4 * hkv:]) == 0, pos
        ratio, ok = R.within(out, y, bound)
        assert ok, (pos, ratio)
        worst = max(worst, ratio)
        if pos >= 2:
            for name, bad in K4.defects(case, exp, pos, cos, sin, S, gs).items():
                if name == "neighbouring group's scale" and gs != 32:
                    continue
                assert not R.within(bad, y, bound)[1], (pos, name)
        del case, c, exp
    print(f"largest err / bound {worst:.3f}")


# ------------------------------------------------------------------------------------------------ harness
_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _model(dtype=torch.float16, kv_pages=None, cache_len=2048, fused=True, gs=64, batch=4, ragged=True, **kw):
    key = (dtype, kv_pages, cache_len, fused, gs, batch, ragged, tuple(sorted(kw.items())))
    if key not in _MODELS:
        m = harness.DecodeModel(SHAPE, dtype=dtype, device=DEV, cache_len=cache_len, fused=fused, seed=11, batch=batch, ragged=ragged, kv_bits=4,
                                kv_group_size=gs, kv_pages=kv_pages, **kw)
        m.capture()
        if kw.get("spec_k"):
            m.capture_spec()
        _MODELS[key] = m
    return _MODELS[key]


def _pair(dtype=torch.float16, cache_len=2048, **kw):
    """The unpaged ragged model and its paged twin (as many pages as the contiguous caches hold)."""
    return _model(dtype, None, cache_len, **kw), _model(dtype, 4 * cache_len // PG, cache_len, **kw)


def _caches(m, b, end):
    out = []
    for blk in m.blocks:
        cv = m.cache_view(blk)
        out += [cv[n][b, :, :end].clone() for n in harness.DecodeModel._CACHE_NAMES]
    return out


def _steps(m, n):
    toks, logits = [], []
    for _ in range(n):
        m.decode()
        toks.append(m.next_tok.clone())
        logits.append(m._bufs["logits"].clone())
    torch.cuda.synchronize(DEV)
    return toks, logits


def _prompts(lengths, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, SHAPE.vocab, (n,), generator=g, device=DEV) for n in lengths]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("dtype,gs", [(torch.float16, 64), (torch.bfloat16, 64), (torch.float16, 32)], ids=["f16-gs64", "bf16-gs64", "f16-gs32"])
def test_kv4_paged_model_equals_unpaged(dtype, gs):
    """Packed prefill of 1, 37, 300 and 1000 tokens, 70 decode() steps across page edges, a refill of slot 2, 20 more steps, then
    release(2) and fork(3, 2) with 10 more steps: tokens, last_logits, step logits and the gathered caches of the paged model equal
    the unpaged model's bit for bit (the unpaged side copies slot 3 into slot 2 for the fork)."""
    prompts, refill = _prompts([1, 37, 300, 1000], 3), _prompts([23], 4)[0]
    runs = []
    for m in _pair(dtype, gs=gs):
        m.reset_state()
        t0 = m.prefill(prompts, chunk=256)
        l0 = m.last_logits.clone()
        a = _steps(m, 70)
        t1 = m.prefill([None, None, refill, None], chunk=16)
        l1 = m.last_logits.clone()
        c = _steps(m, 20)
        assert m.pos.tolist() == [91, 127, 43, 1090]
        if m.kv_pages is not None:
            m.release(2)
            m.fork(3, 2)
        else:
            for blk in m.blocks:
                for n in harness.DecodeModel._CACHE_NAMES:
                    blk[n][2].copy_(blk[n][3])
            m.pos[2].copy_(m.pos[3])
            m.tok[2].copy_(m.tok[3])
        d = _steps(m, 10)
        runs.append((t0, l0, a, t1, l1, c, d, [_caches(m, b, e) for b, e in enumerate(m.pos.tolist())]))
    (t0, l0, a, t1, l1, c, d, ca), (u0, k0, x, u1, k1, y, z, cb) = runs
    assert torch.equal(t0, u0) and torch.equal(l0, k0) and torch.equal(t1, u1) and torch.equal(l1, k1)
    for p, q in ((a, x), (c, y), (d, z)):
        assert _same(p[0], q[0]) and _same(p[1], q[1])
    for p, q in zip(ca, cb):
        assert _same(p, q)


def test_kv4_paged_wrap_equals_unpaged():
    """cache_len 256: slots wrap past the end of the cache and stay equal to the unpaged model."""
    prompts = _prompts([200, 5, 255, 64], 8)
    runs = []
    for m in _pair(torch.float16, cache_len=256):
        m.reset_state()
        t = m.prefill(prompts)
        runs.append((t, _steps(m, 150)))
    assert torch.equal(runs[0][0], runs[1][0]) and _same(runs[0][1][0], runs[1][1][0]) and _same(runs[0][1][1], runs[1][1][1])


def test_kv4_ragged_equal_lengths_equals_lock_step():
    """A ragged batch whose prompts all have the same length equals the lock-step batch bit for bit: prefill tokens, last_logits,
    step tokens and logits."""
    prompt = torch.stack(_prompts([130] * 4, 13))
    runs = []
    for ragged in (True, False):
        m = _model(ragged=ragged)
        m.reset_state()
        t = m.prefill(list(prompt) if ragged else prompt, chunk=64)
        runs.append((t.view(-1), m.last_logits.clone().view(4, -1), _steps(m, 20)))
    (t0, l0, s0), (t1, l1, s1) = runs
    assert torch.equal(t0, t1) and torch.equal(l0, l1) and _same(s0[0], s1[0]) and _same(s0[1], s1[1])


def _state(m):
    st = [m.pos.clone(), m.tok.clone(), m.last_logits.clone()]
    for blk in m.blocks:
        st += [blk[n].clone() for n in harness.DecodeModel._CACHE_NAMES]
    return st


@pytest.mark.parametrize("kv_pages", [None, 128], ids=["contiguous", "paged"])
def test_kv4_score_leaves_prefill_state(kv_pages):
    """score() leaves exactly the state prefill() leaves: positions, tokens, last_logits and every cache tensor."""
    prompts = _prompts([90, 300, 7, 41], 14)
    m = _model(kv_pages=kv_pages)
    m.reset_state()
    m.prefill(prompts, chunk=128)
    a = _state(m)
    m.reset_state()
    lp = m.score(prompts, chunk=128)
    assert len(lp) == 4 and all(torch.isfinite(x).all() for x in lp)
    assert _same(a, _state(m))


def test_kv4_sample_top_k_1_is_greedy():
    """do_sample with top_k=1 draws the greedy stream: prefill tokens and 30 decode steps equal."""
    prompts = _prompts([50, 9, 120, 300], 15)
    runs = []
    for kw in ({}, {"do_sample": True, "top_k": 1, "temperature": 1.0}):
        m = _model(**kw)
        m.reset_state()
        t = m.prefill(prompts)
        runs.append((t, _steps(m, 30)[0]))
    assert torch.equal(runs[0][0], runs[1][0]) and _same(runs[0][1], runs[1][1])


def test_kv4_spec_paged_equals_unpaged():
    """spec_k = 3 over the 4-bit cache, drafts from the prompt lookup on repetitive prompts (self-consistent: they repeat the
    prompt's own continuation): the paged model's emitted tokens, accept counts, positions and caches over 12 verify steps equal the
    unpaged model's bit for bit."""
    base = _prompts([12], 16)[0]
    prompts = [base.repeat(r) for r in (3, 5, 8, 2)]
    runs = []
    for m in _pair(spec_k=3):
        m.reset_state()
        m.prefill(prompts)
        out = []
        for _ in range(12):
            toks, n_new = m.decode_spec()
            out += [toks.clone(), n_new.clone()]
        torch.cuda.synchronize(DEV)
        runs.append((out, [_caches(m, b, e) for b, e in enumerate(m.pos.tolist())], m.pos.tolist()))
    assert _same(runs[0][0], runs[1][0]) and runs[0][2] == runs[1][2]
    for p, q in zip(runs[0][1], runs[1][1]):
        assert _same(p, q)


# The 8-bit cache's logit bars widened by sqrt(255 / 15).  The two paths' k / v rows differ by fp16 / bf16 rounding; where that moves a
# row across a level boundary, the cached element moves by one level.  A 4-bit level is 255 / 15 = 17 times an 8-bit one, and the
# share of elements close enough to a boundary to flip falls by the same factor, so the squared difference of the caches (and of the
# logits it drives) grows 17-fold: the relative L2 by sqrt(17), about 4.1.
FLIP_SCALE = (255 / 15) ** 0.5


def _levels(t):
    return torch.cat([t >> 4, t & 15], dim=-1).to(torch.int16)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_kv4_fused_meets_framework_reference(dtype):
    """fused=5, fused=True and a lock-step batch of 4 against fused=False: the last-position logits of a 1000-token prefill within
    the 8-bit cache's bars times FLIP_SCALE; after 8 more steps fed the reference's tokens, every cache level that differs is off by
    exactly one."""
    tol = (2e-3 if dtype == torch.float16 else 1e-2) * FLIP_SCALE
    for fused, batch in ((5, 1), (True, 1), (True, 4)):
        prompt = torch.randint(0, SHAPE.vocab, (batch, 1000), generator=torch.Generator(device=DEV).manual_seed(batch), device=DEV)
        runs = []
        for f in (fused, False):
            m = _model(dtype, fused=f, batch=batch, ragged=False, cache_len=4096)
            m.reset_state()
            m.prefill(prompt, chunk=256)
            runs.append(m)
        mf, mr = runs
        lf, lr = mf.last_logits.float(), mr.last_logits.float()
        rel = float((lf - lr).norm() / lr.norm())
        print(f"fused={fused} batch={batch}: last-position logits rel L2 {rel:.2e} (bar {tol:.2e})")
        assert rel <= tol, (fused, batch, "prefill", rel)
        # 8 steps, teacher-forced: both models are fed the reference's tokens, so their caches hold the same positions
        for _ in range(8):
            mf.tok.copy_(mr.tok)
            mf.decode(feed_back=False)
            mr.decode()
        torch.cuda.synchronize(DEV)
        end = int(mr.pos.view(-1)[0])
        share = []
        for bf, br in zip(mf.blocks, mr.blocks):
            for side in ("k", "v"):
                a, b = _levels(bf[side + "_cache"][:, :, :end]), _levels(br[side + "_cache"][:, :, :end])
                diff = (a - b).abs()
                assert int(diff.max()) <= 1, (fused, batch, side)
                share.append(float((diff > 0).float().mean()))
        print(f"fused={fused} batch={batch}: share of differing levels {max(share):.4f}")


def test_kv4_prompt_filling_the_cache_wraps_like_a_step():
    """A prompt of exactly cache_len tokens leaves pos at 0, and the next step (which overwrites row 0) gives the reference's token."""
    for fused in (5, True):
        outs = []
        for f in (fused, False):
            m = _model(fused=f, batch=1, ragged=False, cache_len=1024)
            m.reset_state()
            prompt = torch.randint(0, SHAPE.vocab, (1, 1024), generator=torch.Generator(device=DEV).manual_seed(1024), device=DEV)
            tok = m.prefill(prompt, chunk=300)
            assert int(m.pos.item()) == 0
            m.decode()
            torch.cuda.synchronize(DEV)
            assert int(m.pos.item()) == 1
            outs.append((int(tok), int(m.next_tok)))
        assert outs[0] == outs[1], (fused, outs)


@pytest.mark.parametrize("gs", [32, 64])
def test_kv4_cache_bytes_and_arguments(gs):
    """kv_cache_bytes() against the formula (64 level bytes plus scale and zero a row, against 256 bytes in fp16), the kernel name,
    and the arguments the 4-bit cache rejects: a group size outside {32, 64}, or none given."""
    small = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
    m16 = harness.DecodeModel(small, dtype=torch.float16, device=DEV, cache_len=1024, fused=5, seed=3)
    m4 = harness.DecodeModel(small, dtype=torch.float16, device=DEV, cache_len=1024, fused=5, seed=3, kv_bits=4, kv_group_size=gs)
    assert m4.kv_cache_bytes() * 256 == m16.kv_cache_bytes() * (64 + 4 * 128 // gs)
    assert m4.attn_kernel == "split_kv4"
    for kw in ({"kv_group_size": 128}, {"kv_group_size": 16}, {}):
        with pytest.raises(ValueError):
            harness.DecodeModel(small, dtype=torch.float16, device=DEV, cache_len=64, n_layers=1, kv_bits=4, **kw)
