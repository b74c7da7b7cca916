"""Speculative decoding on the H100: the verify attention and the device-position append at the 8B, 70B and tp-8 head shapes up to
position 131071, and DecodeModel(ragged=True, spec_k=K) on a 2-layer Llama-3-8B-shaped model.

Harness: a verify row's logits do not depend on the drafts after it; drafts built from the verify's own targets are all accepted;
the accept count is spec_ref's on the fused path's own logits; the fused verify meets the prefill bars against verify(); a paged
model computes the unpaged model's bits; free-running decode_spec() follows decode()."""
import gc

import pytest
import torch

import attn_split_ref as R
import spec_ref
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

DEV = torch.device("cuda", 0)
SHAPE = harness.LLAMA3_8B
PG = harness.KV_PAGE
K = 3


def test_spec_options_rejected():
    """spec_k without ragged, with do_sample or outside [1, 7] raises ValueError (before any device work)."""
    bad = [dict(spec_k=2), dict(spec_k=2, ragged=True, do_sample=True), dict(spec_k=0, ragged=True), dict(spec_k=8, ragged=True),
           dict(spec_k=2.0, ragged=True)]
    for kw in bad:
        with pytest.raises(ValueError):
            harness.DecodeModel(SHAPE, n_layers=1, device="cpu", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (64, 8), (8, 1)])
def test_verify_kernels_long_context(hq, hkv, dtype):
    """T = 8 rows at positions 131064, 0, 70001, 8191 of a 131072-position cache: the append writes exactly the valid rows (a slot
    at 131064 holds 8), the attention is within spec_ref's bound on every valid element, tickets come back to zero, and the paged
    twins on a scrambled table give the same output bit for bit."""
    lib, code, st = load(), DTYPE_CODE[dtype], stream_ptr(DEV)
    L, T = 131072, 8 if hq // hkv <= 8 else 4
    pos = [L - 8, 0, 70001, 8191]
    B = len(pos)
    g = torch.Generator(device=DEV).manual_seed(hq + hkv)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV).to(dtype)
    q, k, v = rn(B * T, hq * 128), rn(B * T, hkv * 128), rn(B * T, hkv * 128)
    cos, sin = R.tables(L, dtype, DEV)
    kc, vc = rn(B, hkv, L, 128), rn(B, hkv, L, 128)
    p = torch.tensor(pos, dtype=torch.int64, device=DEV)
    qr = torch.zeros(B * T, hq * 128, dtype=dtype, device=DEV)
    check(lib.hqq_b200_glue_rope_append_rows_devpos(ptr(q), ptr(k), ptr(v), ptr(cos), ptr(sin), ptr(kc), ptr(vc), ptr(qr), ptr(p), T, hq, hkv, L, 128, B,
                                                    code, st))
    nbytes = lib.hqq_b200_glue_attn_verify_split_workspace_bytes(hq, hkv, 128, T, B)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    out = torch.zeros(B * T, hq * 128, dtype=dtype, device=DEV)
    check(lib.hqq_b200_glue_attn_verify_split(ptr(qr), ptr(kc), ptr(vc), ptr(p), ptr(out), ptr(ws), hq, hkv, L, 128, T, B, code, st))
    torch.cuda.synchronize(DEV)
    S = R.split_count(torch.cuda.get_device_properties(DEV).multi_processor_count, hkv, L)
    y, bound = spec_ref.verify_reference(qr, kc, vc, pos, T, dtype, S)
    rows = [b * T + t for b in range(B) for t in range(min(T, L - pos[b]))]
    ratio, ok = R.within(out[rows], y[rows], bound[rows])
    assert ok, f"error / bound {ratio:.3f}"
    n_cg = -(-T * (hq // hkv) // 16)
    assert torch.count_nonzero(ws[-4 * B * hkv * n_cg:]) == 0
    # paged twins: every slot's pages in a random physical order
    E = L // PG
    N = B * E
    tab = torch.randperm(N, generator=torch.Generator().manual_seed(1)).view(B, E).to(torch.int32).to(DEV)
    pool = lambda c: torch.cat([c.view(B, hkv, E, PG, 128).permute(0, 2, 1, 3, 4).reshape(N, hkv, PG, 128)[torch.argsort(tab.view(-1).long())],
                                torch.zeros(1, hkv, PG, 128, dtype=dtype, device=DEV)])
    kp, vp = pool(kc), pool(vc)  # the caches after the append, rows in their pages
    kp0, vp0 = kp.clone(), vp.clone()
    qp = torch.zeros_like(qr)
    check(lib.hqq_b200_glue_rope_append_rows_devpos_paged(ptr(q), ptr(k), ptr(v), ptr(cos), ptr(sin), ptr(kp), ptr(vp), ptr(tab), ptr(qp), ptr(p), T, hq,
                                                          hkv, L, 128, B, N, code, st))
    outp = torch.zeros_like(out)
    check(lib.hqq_b200_glue_attn_verify_split_paged(ptr(qp), ptr(kp), ptr(vp), ptr(tab), ptr(p), ptr(outp), ptr(ws), hq, hkv, L, 128, T, B, N, code, st))
    torch.cuda.synchronize(DEV)
    assert torch.equal(kp, kp0) and torch.equal(vp, vp0)  # the same rows rewritten with the same bits
    assert torch.equal(qp[rows], qr[rows]) and torch.equal(outp[rows], out[rows])


# ------------------------------------------------------------------------------------------------------------------ harness
_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    """The models (and their captured graphs) live for this module only: the suite runs in one process."""
    yield
    _MODELS.clear()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _model(dtype, kv_pages=None, cache_len=2048, fused=True, batch=4, kv_bits=16):
    key = (dtype, kv_pages, cache_len, fused, batch, kv_bits)
    if key not in _MODELS:
        m = harness.DecodeModel(SHAPE, n_layers=2, dtype=dtype, device=DEV, cache_len=cache_len, fused=fused, seed=11, batch=batch, ragged=True,
                                kv_pages=kv_pages, spec_k=K, kv_bits=kv_bits)
        if fused:
            m.capture()
            m.capture_spec()
        _MODELS[key] = m
    return _MODELS[key]


def _prompts(lengths, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, 50, (n,), generator=g, device=DEV) for n in lengths]  # a small alphabet: prompt lookup finds matches


def _save(m):
    s = [t.clone() for t in (m.pos, m.tok, m.next_tok, m.hist)]
    if m.kv_pages is not None:
        pa = m.pages
        s.append(([r[:] for r in pa.table], pa.ref[:], pa.free[:], pa.pos[:], pa.active[:], m.page_table.clone()))
    return s


def _restore(m, s):
    for t, v in zip((m.pos, m.tok, m.next_tok, m.hist), s):
        t.copy_(v)
    if m.kv_pages is not None:
        pa = m.pages
        tb, ref, free, pos, act, dt = s[4]
        pa.table, pa.ref, pa.free, pa.pos, pa.active = [r[:] for r in tb], ref[:], free[:], pos[:], act[:]
        m.page_table.copy_(dt)


def _spec(m, drafts=None):
    tok, n_new = m.decode_spec(drafts)
    return tok, n_new, m.spec_logits.clone()


F16, BF16 = torch.float16, torch.bfloat16
# (dtype, kv_pages, kv_bits, batch)
CFGS = [(F16, None, 16, 4), (BF16, None, 16, 4), (F16, 512, 16, 4), (BF16, 512, 16, 4), (F16, None, 8, 4), (BF16, None, 8, 4), (F16, 512, 8, 4),
        (BF16, 512, 8, 4), (F16, None, 16, 1), (BF16, 512, 16, 1), (F16, None, 8, 1), (BF16, 512, 8, 1)]
CFG_IDS = [f"{'f16' if d == F16 else 'bf16'}-kv{kb}-b{b}" + ("-paged" if p else "") for d, p, kb, b in CFGS]
PROMPTS = [5, 37, 300, 1000]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,kv_pages,kv_bits,batch", CFGS, ids=CFG_IDS)
def test_spec_prefix_invariance_and_self_consistent_drafts(dtype, kv_pages, kv_bits, batch):
    """Row r's logits and target do not change by a bit when the drafts after r change; drafts built one verify at a time from the
    verify's own targets are all accepted, and the emitted tokens are those targets plus t_K; the accept count equals spec_ref's on
    the fused path's own logits."""
    m = _model(dtype, kv_pages, batch=batch, kv_bits=kv_bits)
    m.reset_state()
    m.prefill(_prompts(PROMPTS[-batch:], 3), chunk=256)
    st = _save(m)
    B = m.batch
    d = torch.full((B, K), -1, dtype=torch.long, device=DEV)
    rows = []
    for r in range(K + 1):  # verify r: drafts d1 .. dr from the earlier targets, the rest -1
        _restore(m, st)
        _, n_new, lg = _spec(m, d)
        rows.append(lg)
        tg = lg.argmax(-1)
        assert torch.equal(tg, m._spec_targets.view(B, K + 1))
        if r < K:
            d[:, r] = tg[:, r]
        for rr in range(r + 1):  # rows <= r saw the same inputs in every earlier verify
            assert torch.equal(lg[:, rr], rows[rr][:, rr])
    assert n_new.tolist() == [K + 1] * B
    tok = m._spec_tokens
    assert torch.equal(tok[:, :K], d) and torch.equal(tok[:, K], rows[-1].argmax(-1)[:, K])
    # random drafts: the accept count is spec_ref's on the logits
    _restore(m, st)
    pos0, tok0 = m.pos.tolist(), m.tok.tolist()
    dr = torch.where(torch.rand(B, K, device=DEV) < 0.5, d, torch.randint(0, 50, (B, K), device=DEV))
    toks, n_new, lg = _spec(m, dr)
    tg = lg.argmax(-1).tolist()
    for b in range(B):
        em, a, p = spec_ref.accept(tok0[b], dr[b].tolist(), tg[b], pos0[b], m.cache_len)
        assert int(n_new[b]) == a + 1 and toks[b, :a + 1].tolist() == em and int(m.pos[b]) == p


@pytest.mark.gpu
@pytest.mark.parametrize("kv_bits", [16, 8], ids=["kv16", "kv8"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_spec_fused_meets_reference(dtype, kv_bits):
    """Teacher-forced verify logits of the fused path against verify() (fused=False) from one state -- the fused prefill's caches and
    positions copied into the reference model, one next token and one set of drafts -- within the prefill bars (relative L2 2e-3
    fp16, 1e-2 bf16; with the 8-bit cache the ragged prefill's 5e-3 fp16 bar, where a new row's 8-bit level can flip between the two
    paths' k rows).  The rows the verify wrote into the caches agree within one quantisation step (8-bit) or 1e-2 relative.  (Each model's own prefill would add the two prefill paths' difference, which on this model already reaches
    1.1e-2 in bf16: DESIGN.md 3.5.)"""
    tol = (2e-3 if kv_bits == 16 else 5e-3) if dtype == torch.float16 else 1e-2
    prompts = _prompts([5, 37, 300, 1000], 4)
    g = torch.Generator(device=DEV).manual_seed(9)
    d = torch.randint(0, 50, (4, K), device=DEV, generator=g)
    tok = torch.randint(0, 50, (4,), device=DEV, generator=g)
    mf = _model(dtype, fused=True, kv_bits=kv_bits)
    mf.reset_state()
    mf.prefill(prompts, chunk=256)
    pos = mf.pos.clone()
    out, rows = [], []
    for fused in (True, False):
        m = _model(dtype, fused=fused, kv_bits=kv_bits)
        if not fused:
            m.reset_state()
            for bf, br in zip(mf.blocks, m.blocks):
                for n in harness.DecodeModel._CACHE_NAMES:
                    if n in bf:
                        br[n].copy_(bf[n])
        m.pos.copy_(pos)
        m.tok.copy_(tok)
        m._spec_drafts.copy_(d)
        with torch.no_grad():
            (m.spec_graph.replay if fused else m.verify)()
        out.append(m.spec_logits.float().clone())
        blk = m.blocks[-1]
        if kv_bits == 8:
            kc = harness.kv8_dequantize(blk["k_cache"], blk["k_scale"], blk["k_zero"])
        else:
            kc = blk["k_cache"]
        rows.append(torch.stack([kc[b, :, int(pos[b]):int(pos[b]) + K + 1].float() for b in range(4)]))
    rel = float((out[0] - out[1]).norm() / out[1].norm())
    assert rel <= tol, rel
    if kv_bits == 8:  # at most one level apart: |diff| <= the row's scale
        step = torch.stack([mf.blocks[-1]["k_scale"][b, :, int(pos[b]):int(pos[b]) + K + 1].float() for b in range(4)]).amax()
        ulp = 2.0 ** -(10 if dtype == torch.float16 else 7) * float(rows[1].abs().max())  # plus one rounding of the dequantised value
        assert float((rows[0] - rows[1]).abs().max()) <= 1.05 * float(step) + ulp
    else:
        assert float((rows[0] - rows[1]).norm() / rows[1].norm()) <= 1e-2


PAGED_CFGS = [(F16, 16, 4), (BF16, 16, 4), (F16, 8, 4), (BF16, 8, 4), (F16, 16, 1), (BF16, 8, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,kv_bits,batch", PAGED_CFGS, ids=[f"{'f16' if d == F16 else 'bf16'}-kv{kb}-b{b}" for d, kb, b in PAGED_CFGS])
def test_spec_paged_equals_unpaged(dtype, kv_bits, batch):
    """Packed prefill of 1, 37, 300 and 1000 tokens, 30 decode_spec() calls with prompt-lookup drafts, a refill of slot 2, interleaved
    decode() steps, then (paged) release and fork against the unpaged model with the slot copied: tokens, n_new, logits and gathered
    caches bit for bit.  At batch 1: the prefill of 300 tokens, the refill of slot 0, no release / fork."""
    runs = []
    names = [n for n in harness.DecodeModel._CACHE_NAMES if kv_bits == 8 or n in ("k_cache", "v_cache")]
    for kv_pages in (None, 512):
        m = _model(dtype, kv_pages, batch=batch, kv_bits=kv_bits)
        m.reset_state()
        rec = [m.prefill(_prompts([1, 37, 300, 1000] if batch == 4 else [300], 5), chunk=256)]
        for i in range(30):
            rec += list(_spec(m))
        refill = [None] * batch
        refill[min(2, batch - 1)] = _prompts([23], 6)[0]
        rec.append(m.prefill(refill, chunk=16))
        for i in range(6):
            if i % 2:
                m.decode()
                rec.append(m.next_tok.clone())
            else:
                rec += list(_spec(m))
        if batch == 1:
            pass
        elif kv_pages is None:
            for blk in m.blocks:
                for n in names:
                    blk[n][1].copy_(blk[n][3])
            m.pos[1].copy_(m.pos[3])
            m.tok[1].copy_(m.tok[3])
            m.hist[1].copy_(m.hist[3])
        else:
            m.release(1)
            m.fork(3, 1)
        for i in range(4):
            rec += list(_spec(m))
        torch.cuda.synchronize(DEV)
        ends = m.pos.tolist()
        caches = [m.cache_view(blk)[n][b, :, :ends[b]].clone() for blk in m.blocks for n in names for b in range(m.batch) if b != 1 or batch == 1]
        runs.append((rec, caches, ends))
    (ra, ca, ea), (rb, cb, eb) = runs
    assert ea == eb
    assert len(ra) == len(rb) and all(torch.equal(x, y) for x, y in zip(ra, rb))
    assert all(torch.equal(x, y) for x, y in zip(ca, cb))


@pytest.mark.gpu
def test_spec_refill_leaves_other_slots_alone():
    """Refilling slot 2 between decode_spec() calls leaves slots 0, 1 and 3's tokens and logits bit for bit as in a run without it."""
    runs = []
    for refill in (False, True):
        m = _model(torch.float16)
        m.reset_state()
        m.prefill(_prompts([9, 37, 300, 100], 7), chunk=256)
        rec = []
        for i in range(10):
            if i == 4 and refill:
                m.prefill([None, None, _prompts([50], 8)[0], None])
            t, n, lg = _spec(m)
            rec.append((t[[0, 1, 3]], n[[0, 1, 3]], lg[[0, 1, 3]]))
        runs.append(rec)
    for x, y in zip(*runs):
        assert all(torch.equal(a, b) for a, b in zip(x, y))


@pytest.mark.gpu
@pytest.mark.parametrize("kv_pages", [None, 8], ids=["contiguous", "paged"])
def test_spec_cache_end_clamps_and_wraps(kv_pages):
    """cache_len 256, prompts ending at 250 .. 253: every window is clamped to the cache and positions wrap to 0 by the rule."""
    m = _model(torch.float16, kv_pages=kv_pages, cache_len=256, batch=2)
    m.reset_state()
    m.prefill(_prompts([250, 253], 9))
    for _ in range(6):
        pos0 = m.pos.tolist()
        _, n_new = m.decode_spec()
        for b in range(2):
            assert 1 <= int(n_new[b]) <= min(K + 1, 256 - pos0[b])
            assert int(m.pos[b]) == (pos0[b] + int(n_new[b])) % 256
    assert max(m.pos.tolist()) < 250  # both wrapped


@pytest.mark.gpu
@pytest.mark.parametrize("kv_bits,batch", [(16, 4), (16, 1), (8, 4), (8, 1)], ids=["kv16-b4", "kv16-b1", "kv8-b4", "kv8-b1"])
def test_spec_follows_plain_decode(kv_bits, batch):
    """Free-running greedy tokens from decode_spec() against decode() from the same state: the first tokens agree, and all but at most
    two of 24 -- or, where a stream leaves decode()'s, decode()'s own logits at that step hold the two tokens within 1 % of the
    row's largest magnitude: a near tie that the verify pass's different rounding (M = batch (K + 1) rows; with the 8-bit cache, a
    new row's level) may break the other way, after which both streams are valid greedy continuations.  (At batch 1 decode() picks
    with the argmax kernel and the verify with torch.argmax: first index on ties both.)"""
    m = _model(torch.float16, batch=batch, kv_bits=kv_bits)
    m.reset_state()
    m.prefill(_prompts([40, 80, 120, 160][:batch], 10), chunk=256)
    st = _save(m)
    plain, logits = [], []
    for _ in range(24):
        plain.append(m.tok.clone())
        m.decode()
        logits.append(m._bufs["logits"].float().clone())
    plain = torch.stack(plain, 1)
    _restore(m, st)
    spec = [[int(m.tok[b])] for b in range(m.batch)]
    while min(len(s) for s in spec) < 24:
        toks, n_new = m.decode_spec()
        for b in range(m.batch):
            spec[b] += toks[b, :int(n_new[b])].tolist()
    for b in range(m.batch):
        got = torch.tensor(spec[b][:24], device=DEV)
        assert got[:2].tolist() == plain[b, :2].tolist()
        miss = (got != plain[b]).nonzero().view(-1).tolist()
        if len(miss) <= 2:
            continue
        i = miss[0]  # token i is the pick of step i - 1
        lg = logits[i - 1][b]
        gap = float(lg[int(plain[b, i])] - lg[int(got[i])])
        assert 0 <= gap <= 0.01 * float(lg.abs().max()), (b, i, gap, float(lg.abs().max()))
