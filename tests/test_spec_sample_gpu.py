"""Sampled speculative decoding on the H100: hqq_b200_glue_sample_pos at the full vocabulary, and DecodeModel(do_sample=True,
sample_keys="position", spec_k=K) on a 2-layer Llama-3-8B-shaped model.

Kernel tokens are held to tests/sample_ref.py's rule against sample_tokens with the rows' position keys; a chi-square test of 2^20
draws over the sequence number checks the distribution.  Harness: every fused token (prefill, decode, verify) is the restatement's
token on the fused path's own logits at its slot, position and sequence number; a refill leaves the other slots' streams alone; a
reset reproduces a run; the accept count is spec_ref's on the verify's own targets; top_k = 1 reproduces greedy speculative
decoding; paged equals unpaged bit for bit; the fused verify and free-running decode_spec() agree with the references up to the
two paths' logit differences."""
import gc

import pytest
import torch

import sample_ref as S
import spec_ref
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SHAPE = harness.LLAMA3_8B
V = SHAPE.vocab
K = 3
SEED = 0x5EED_5A3B_1E50_0F00
# the reference generator's sampling defaults
SAMPLE = dict(do_sample=True, sample_keys="position", temperature=0.6, top_k=5, top_p=1.0, sample_seed=21)


def sample_pos(x, T, temp, k, p, pos, seq, seed=SEED):
    rows = x.shape[0]
    pt, st = torch.tensor(pos, dtype=torch.int64, device=DEV), torch.tensor(seq, dtype=torch.int64, device=DEV)
    out = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
    check(load().hqq_b200_glue_sample_pos(ptr(x), V, x.stride(0), rows, temp, k, p, seed, T, ptr(pt), ptr(st), ptr(out), DTYPE_CODE[x.dtype],
                                          stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out


def held(lg, temp, k, p, seed, pos, seq):
    """Per row of lg [B, V] (row b = slot b): (float64 token, the tokens the kernel may return) under position keys."""
    ctr = harness.position_counter(torch.as_tensor(pos).view(-1).cpu(), torch.as_tensor(seq).view(-1).cpu())
    u = harness.philox_uniforms(V, lg.shape[0], seed, ctr)
    return [(t0, ok) for t0, ok, _ in S.accepted(lg.cpu(), temp, k, p, u)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_sample_pos_full_vocab_matches_float64(dtype):
    g = torch.Generator(device=DEV).manual_seed(DTYPE_CODE[dtype])
    pos, seq = [63, 131071], [1, 2 ** 31 - 1]
    differ = rows = 0
    for T, temp, k, p in ((1, 0.6, 5, 1.0), (4, 1.0, 0, 0.9), (8, 0.7, 50, 0.95)):
        x = (torch.randn(2 * T, V + 64, generator=g, device=DEV) * 2.5).to(dtype)
        got = sample_pos(x, T, temp, k, p, pos, seq).view(2, T).cpu()
        for t in range(T):
            for b, (t0, ok) in enumerate(held(x.view(2, T, -1)[:, t, :V], temp, k, p, SEED, [q + t for q in pos], seq)):
                assert int(got[b, t]) in ok, (T, t, b, int(got[b, t]), t0)
                differ += int(got[b, t]) != t0
                rows += 1
    print(f"{dtype}: {differ} of {rows} rows differ from float64 (within the allowed set)")


def test_sample_pos_chi_square_over_seq():
    """2^20 draws from one fixed row: 4096 slots per launch, seq 0 .. 255; the counts match the kept softmax."""
    from scipy.stats import chisquare
    gen = torch.Generator().manual_seed(2024)
    row = torch.randn(V, generator=gen, dtype=torch.float64) * 1.5
    row[torch.randperm(V, generator=gen)[:64]] += torch.linspace(3.0, 9.0, 64, dtype=torch.float64)
    row = row.to(torch.float16)
    R, C = 4096, 256
    for temp, k, p in ((0.6, 5, 1.0), (1.0, 0, 0.9)):
        x = row.to(DEV).view(1, V).expand(R, V).contiguous()
        pos = torch.full((R,), 777, dtype=torch.int64, device=DEV)
        seq = torch.zeros(R, dtype=torch.int64, device=DEV)
        out = torch.empty(R, dtype=torch.int64, device=DEV)
        counts = torch.zeros(V, dtype=torch.int64, device=DEV)
        for c in range(C):
            seq.fill_(c)
            check(load().hqq_b200_glue_sample_pos(ptr(x), V, V, R, temp, k, p, SEED, 1, ptr(pos), ptr(seq), ptr(out), DTYPE_CODE[torch.float16],
                                                  stream_ptr(DEV)))
            counts += torch.bincount(out, minlength=V)
        counts = counts.cpu().double()
        lv = row.double().view(1, V)
        keep = S.keep_topp(lv, S.keep_topk(lv, k), S.fp32(temp), S.fp32(p))[0]
        w = torch.where(keep, torch.exp((lv[0] - lv[0].max()) / S.fp32(temp)), torch.zeros(V, dtype=torch.float64))
        exp = w / w.sum() * (R * C)
        assert counts[~keep].sum() == 0, "a draw outside the kept set"
        big = exp >= 5
        obs, ex = torch.cat([counts[big], counts[~big].sum().view(1)]), torch.cat([exp[big], exp[~big].sum().view(1)])
        if ex[-1] == 0:
            obs, ex = obs[:-1], ex[:-1]
        stat, pval = chisquare(obs.numpy(), ex.numpy())
        print(f"T {temp} top_k {k} top_p {p}: kept {int(keep.sum())}, chi2 {stat:.1f}, p {pval:.3g}")
        assert pval >= 1e-6


# ------------------------------------------------------------------------------------------------------------------ harness
_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _drop_models()


def _drop_models():
    _MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _model(dtype=torch.float16, kv_pages=None, batch=4, kv_bits=16, fused=True, ragged=True, spec=True, **kw):
    opts = dict(SAMPLE, **kw)
    key = (dtype, kv_pages, batch, kv_bits, fused, ragged, spec, tuple(sorted(opts.items())))
    if key not in _MODELS:
        m = harness.DecodeModel(SHAPE, n_layers=2, dtype=dtype, device=DEV, cache_len=2048, fused=fused, seed=11, batch=batch, ragged=ragged,
                                kv_pages=kv_pages, spec_k=K if spec else None, kv_bits=kv_bits, kv_group_size=64 if kv_bits == 4 else None,
                                **opts)
        if fused:
            m.capture()
            if spec:
                m.capture_spec()
        _MODELS[key] = m
    return _MODELS[key]


def _prompts(lengths, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, 50, (n,), generator=g, device=DEV) for n in lengths]  # a small alphabet: prompt lookup finds matches


def _save(m):
    s = [t.clone() for t in (m.pos, m.tok, m.next_tok, m.hist, m.seq)]
    if m.kv_pages is not None:
        pa = m.pages
        s.append(([r[:] for r in pa.table], pa.ref[:], pa.free[:], pa.pos[:], pa.active[:], m.page_table.clone()))
    return s


def _restore(m, s):
    for t, v in zip((m.pos, m.tok, m.next_tok, m.hist, m.seq), s):
        t.copy_(v)
    if m.kv_pages is not None:
        pa = m.pages
        tb, ref, free, pos, act, dt = s[5]
        pa.table, pa.ref, pa.free, pa.pos, pa.active = [r[:] for r in tb], ref[:], free[:], pos[:], act[:]
        m.page_table.copy_(dt)


def _spec(m, drafts=None):
    tok, n_new = m.decode_spec(drafts)
    return tok, n_new, m.spec_logits.clone()


def _check_tokens(lg, toks, pos, seq, m):
    for b, (t0, ok) in enumerate(held(lg, m.temperature, m.top_k, m.top_p, m.sample_seed, pos, seq)):
        assert int(toks[b]) in ok, (b, int(toks[b]), t0, pos, seq)


@pytest.mark.parametrize("ragged,batch,fused", [(True, 4, True), (False, 4, True), (False, 1, 5)], ids=["ragged", "lockstep", "fused5"])
def test_fused_tokens_are_the_position_keyed_draws(ragged, batch, fused):
    """Prefill's token and every decode() token against sample_tokens at the row's slot, position and seq, on the fused path's own
    logits.  A second prefill from position 0 counts a new sequence in every slot; a reset and re-run reproduce the stream."""
    m = _model(batch=batch, ragged=ragged, fused=fused, spec=ragged)
    runs = []
    for _ in range(2):
        m.reset_state()
        m.prefill(torch.stack(_prompts([30] * batch, 3)) if not ragged else _prompts([30, 5, 60, 17], 3), chunk=64)
        m.prefill(torch.stack(_prompts([30] * batch, 4)) if not ragged else _prompts([30, 5, 60, 17], 4), chunk=64)
        assert m.seq.tolist() == [2] * batch
        last = [29] * batch if not ragged else [29, 4, 59, 16]
        rec = [m.tok.clone()]
        _check_tokens(m.last_logits, m.tok, last, m.seq, m)
        for _ in range(8):
            pos = m.pos.expand(batch).clone()
            m.decode()
            _check_tokens(m._bufs["logits"], m.next_tok, pos, m.seq, m)
            rec.append(m.next_tok.clone())
        runs.append(torch.stack(rec))
    assert torch.equal(runs[0], runs[1])


@pytest.mark.parametrize("spec", [False, True], ids=["decode", "decode_spec"])
def test_refill_leaves_other_slots_alone(spec):
    """Refilling slot 2 leaves slots 0, 1 and 3's sampled tokens (and logits) bit for bit as in a run without it."""
    m = _model()
    runs = []
    for refill in (False, True):
        m.reset_state()
        m.prefill(_prompts([9, 37, 300, 100], 7), chunk=256)
        rec = []
        for i in range(10):
            if i == 4 and refill:
                m.prefill([None, None, _prompts([50], 8)[0], None])
            if spec:
                t, n, lg = _spec(m)
                rec.append((t[[0, 1, 3]], n[[0, 1, 3]], lg[[0, 1, 3]]))
            else:
                m.decode()
                rec.append((m.next_tok[[0, 1, 3]].clone(), m._bufs["logits"][[0, 1, 3]].clone()))
        runs.append(rec)
    for x, y in zip(*runs):
        assert all(torch.equal(a, b) for a, b in zip(x, y))


def test_verify_targets_accept_and_self_consistent_drafts():
    """The verify's targets are the position-keyed draws from its own logits rows, the accept count is spec_ref's on them, and
    drafts built one verify at a time from the verify's own targets are all accepted."""
    m = _model()
    m.reset_state()
    m.prefill(_prompts([5, 37, 300, 1000], 3), chunk=256)
    st = _save(m)
    B, T = m.batch, K + 1
    d = torch.full((B, K), -1, dtype=torch.long, device=DEV)
    for r in range(T):
        _restore(m, st)
        pos0, tok0 = m.pos.tolist(), m.tok.tolist()
        toks, n_new, lg = _spec(m, d)
        tg = m._spec_targets.view(B, T).clone()
        for t in range(T):
            _check_tokens(lg[:, t], tg[:, t], [p + t for p in pos0], m.seq, m)
        for b in range(B):
            em, a, p = spec_ref.accept(tok0[b], d[b].tolist(), tg[b].tolist(), pos0[b], m.cache_len)
            assert int(n_new[b]) == a + 1 and toks[b, :a + 1].tolist() == em and int(m.pos[b]) == p
        if r < K:
            d[:, r] = tg[:, r]
    assert n_new.tolist() == [T] * B
    # random drafts around the targets
    _restore(m, st)
    pos0, tok0 = m.pos.tolist(), m.tok.tolist()
    dr = torch.where(torch.rand(B, K, device=DEV) < 0.5, d, torch.randint(0, 50, (B, K), device=DEV))
    toks, n_new, lg = _spec(m, dr)
    tg = m._spec_targets.view(B, T).tolist()
    for b in range(B):
        em, a, p = spec_ref.accept(tok0[b], dr[b].tolist(), tg[b], pos0[b], m.cache_len)
        assert int(n_new[b]) == a + 1 and toks[b, :a + 1].tolist() == em


def test_top_k_1_reproduces_greedy_spec():
    """With top_k = 1 the sampled decode_spec() stream is the greedy one, verify by verify, except at an exactly tied maximum (every
    tied element stays in the race there): such a slot's stream may part, and is not followed further."""
    mg = harness.DecodeModel(SHAPE, n_layers=2, dtype=torch.float16, device=DEV, cache_len=2048, seed=11, batch=4, ragged=True, spec_k=K)
    mg.capture()
    mg.capture_spec()
    ms = _model(top_k=1)
    for m in (mg, ms):
        m.reset_state()
        m.prefill(_prompts([40, 80, 120, 160], 10), chunk=256)
    assert torch.equal(mg.tok, ms.tok)
    live = [True] * 4
    for _ in range(12):
        tg, ng, lgg = _spec(mg)
        ts, ns, _ = _spec(ms)
        for b in range(4):
            if live[b] and not torch.equal(tg[b], ts[b]):  # both verified the same window: row i's logits are the same
                i = int((tg[b] != ts[b]).nonzero()[0])
                row = lgg[b, i].float()
                assert row[int(ts[b, i])] == row.max() and row[int(tg[b, i])] == row.max(), (b, i)
                live[b] = False
    assert sum(live) >= 2, live
    del mg
    gc.collect()


F16, BF16 = torch.float16, torch.bfloat16
MATRIX = [(d, kb, b) for d in (F16, BF16) for kb in (16, 8, 4) for b in (4, 1)]


@pytest.mark.parametrize("dtype,kv_bits,batch", MATRIX, ids=[f"{'f16' if d == F16 else 'bf16'}-kv{kb}-b{b}" for d, kb, b in MATRIX])
def test_sampled_spec_paged_equals_unpaged(dtype, kv_bits, batch):
    """test_spec_paged_equals_unpaged's sequence, sampled: packed prefill, 20 decode_spec() calls, a refill, interleaved decode()
    steps, then (paged) release and fork against the unpaged model with the slot (and its seq) copied: tokens, n_new, logits and
    gathered caches bit for bit."""
    _drop_models()
    runs = []
    names = [n for n in harness.DecodeModel._CACHE_NAMES if kv_bits != 16 or n in ("k_cache", "v_cache")]
    for kv_pages in (None, 512):
        m = _model(dtype, kv_pages, batch=batch, kv_bits=kv_bits)
        m.reset_state()
        rec = [m.prefill(_prompts([1, 37, 300, 1000] if batch == 4 else [300], 5), chunk=256)]
        for _ in range(20):
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
        if batch == 4 and kv_pages is None:
            for blk in m.blocks:
                for n in names:
                    blk[n][1].copy_(blk[n][3])
            for t in (m.pos, m.tok, m.hist, m.seq):
                t[1].copy_(t[3])
        elif batch == 4:
            m.release(1)
            m.fork(3, 1)
        for _ in range(4):
            rec += list(_spec(m))
        rec.append(m.seq.clone())
        torch.cuda.synchronize(DEV)
        ends = m.pos.tolist()
        caches = [m.cache_view(blk)[n][b, :, :ends[b]].clone() for blk in m.blocks for n in names for b in range(m.batch) if b != 1 or batch == 1]
        runs.append((rec, caches, ends))
    _drop_models()
    (ra, ca, ea), (rb, cb, eb) = runs
    assert ea == eb
    assert len(ra) == len(rb) and all(torch.equal(x, y) for x, y in zip(ra, rb))
    assert all(torch.equal(x, y) for x, y in zip(ca, cb))


def _near(lg, x, y, margin, temp, k, p, seed, pos, seq):
    """Tokens x, y of one row lg [V] (float64 on the CPU) are a near tie: their perturbed keys within `margin`, or one of them
    within `margin` times T of the top-k pivot or the top-p threshold."""
    ctr = harness.position_counter(torch.tensor([pos]), torch.tensor([seq]))
    u = harness.philox_uniforms(V, 1, seed, ctr)[0]
    key = lg / S.fp32(temp) - torch.log(-torch.log(u))
    if abs(float(key[x] - key[y])) <= margin:
        return True
    lv = lg.view(1, V)
    keep_k = S.keep_topk(lv, k)
    edges = [float(lv[keep_k].min()), float(lv[S.keep_topp(lv, keep_k, S.fp32(temp), S.fp32(p))].min())]
    return any(abs(float(lg[t]) - e) <= margin * S.fp32(temp) for t in (x, y) for e in edges)


@pytest.mark.parametrize("kv_bits", [16, 8], ids=["kv16", "kv8"])
def test_fused_verify_meets_reference(kv_bits):
    """From one state (the fused prefill's caches, positions and seq copied into the fused=False model, one token and one set of
    drafts), the fused verify's targets equal verify()'s, except where the two tokens' float64 perturbed keys lie within twice the
    row's largest logit difference between the paths over T (or one token sits that close to the top-k / top-p edge)."""
    prompts = _prompts([5, 37, 300, 1000], 4)
    g = torch.Generator(device=DEV).manual_seed(9)
    d = torch.randint(0, 50, (4, K), device=DEV, generator=g)
    tok = torch.randint(0, 50, (4,), device=DEV, generator=g)
    mf = _model(kv_bits=kv_bits)
    mf.reset_state()
    mf.prefill(prompts, chunk=256)
    pos, seq = mf.pos.clone(), mf.seq.clone()
    out = []
    for fused in (True, False):
        m = _model(kv_bits=kv_bits, fused=fused)
        if not fused:
            m.reset_state()
            for bf, br in zip(mf.blocks, m.blocks):
                for n in harness.DecodeModel._CACHE_NAMES:
                    if n in bf:
                        br[n].copy_(bf[n])
        m.pos.copy_(pos)
        m.seq.copy_(seq)
        m.tok.copy_(tok)
        m._spec_drafts.copy_(d)
        with torch.no_grad():
            (m.spec_graph.replay if fused else m.verify)()
        out.append((m.spec_logits.double().cpu().clone(), m._spec_targets.view(4, K + 1).cpu().clone()))
    (lf, tf), (lr, tr) = out
    differ = 0
    for b in range(4):
        for t in range(K + 1):
            x, y = int(tf[b, t]), int(tr[b, t])
            if x != y:
                differ += 1
                dl = float((lf[b, t] - lr[b, t]).abs().max())
                assert _near(lf[b, t], x, y, 2 * dl / S.fp32(SAMPLE["temperature"]), SAMPLE["temperature"], SAMPLE["top_k"], SAMPLE["top_p"],
                             SAMPLE["sample_seed"], int(pos[b]) + t, int(seq[b])), (b, t, x, y, dl)
    print(f"kv{kv_bits}: {differ} of {4 * (K + 1)} targets differ")


@pytest.mark.parametrize("kv_bits,batch", [(16, 4), (16, 1), (8, 4), (4, 1)], ids=["kv16-b4", "kv16-b1", "kv8-b4", "kv4-b1"])
def test_sampled_spec_follows_plain_decode(kv_bits, batch):
    """Free-running sampled decode_spec() against position-keyed decode() from the same state: a slot's streams agree up to their
    first divergence, and there decode()'s own perturbed keys hold the two tokens within 1 % of the row's largest magnitude over T,
    or one of them sits on the top-k / top-p edge within that margin: a near tie that the verify pass's different rounding may break
    the other way, after which both streams are valid samples."""
    m = _model(batch=batch, kv_bits=kv_bits)
    m.reset_state()
    m.prefill(_prompts([40, 80, 120, 160][:batch], 10), chunk=256)
    st = _save(m)
    plain, logits, poss = [], [], []
    for _ in range(24):
        plain.append(m.tok.clone())
        poss.append(m.pos.clone())
        m.decode()
        logits.append(m._bufs["logits"].double().cpu().clone())
    plain = torch.stack(plain, 1)
    _restore(m, st)
    spec = [[int(m.tok[b])] for b in range(batch)]
    while min(len(s) for s in spec) < 24:
        toks, n_new = m.decode_spec()
        for b in range(batch):
            spec[b] += toks[b, :int(n_new[b])].tolist()
    T = S.fp32(SAMPLE["temperature"])
    for b in range(batch):
        got = torch.tensor(spec[b][:24], device=DEV)
        miss = (got != plain[b]).nonzero().view(-1).tolist()
        if not miss:
            continue
        i = miss[0]  # token i is the pick of step i - 1
        lg = logits[i - 1][b]
        assert _near(lg, int(plain[b, i]), int(got[i]), 0.01 * float(lg.abs().max()) / T, SAMPLE["temperature"], SAMPLE["top_k"],
                     SAMPLE["top_p"], SAMPLE["sample_seed"], int(poss[i - 1][b]), int(m.seq[b])), (b, i)
