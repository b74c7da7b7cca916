"""Paged KV cache on the H100: the _paged entry points (csrc/decode_glue.cu) at the 8B, 70B and tp-8 head shapes, and
DecodeModel(ragged=True, kv_pages=N) on a 2-layer Llama-3-8B-shaped model.

Kernels: each _paged launch equals its contiguous ragged counterpart run on the cache gathered through a scrambled table, bit for
bit.  Harness: the same sequence of calls on the paged and the unpaged ragged model gives equal tokens, logits and caches, bit for
bit; a fork equals the unpaged model with slot 0's cache copied into the other slots."""
import ctypes
import gc

import pytest
import torch

import attn_split_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
HEADS = [(32, 8), (64, 8), (8, 1)]
PG = harness.KV_PAGE


def ints(xs):
    return (ctypes.c_int * len(xs))(*xs)


def table(ends, entries, seed):
    """Scrambled table: slot b owns pages for positions [0, ends[b]) in a random physical order, slot b > 0 shares slot b - 1's first
    page when both hold more than one page; other entries are the sink."""
    need = [-(-e // PG) for e in ends]
    N = sum(need) + 2
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(seed)).tolist()
    tab = torch.full((len(ends), entries), N, dtype=torch.int32)
    k = 0
    for b, n in enumerate(need):
        tab[b, :n] = torch.tensor(perm[k:k + n], dtype=torch.int32)
        k += n
    for b in range(1, len(ends)):
        if need[b] > 1 and need[b - 1] > 1:
            tab[b, 0] = tab[b - 1, 0]
    return tab.to(DEV), N


def gather(pool, tab):
    B, E = tab.shape
    return pool[tab.long()].permute(0, 2, 1, 3, 4).reshape(B, pool.shape[1], E * PG, pool.shape[3]).contiguous()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
@pytest.mark.parametrize("kind", ["batch", "split", "kv8"])
def test_paged_decode_equals_seqpos_on_gathered_cache(kind, hq, hkv, dtype):
    """Positions up to 8191 (single kernel) and 131071 (split, kv8) over a scrambled table: output, tickets and every written row
    equal the _seqpos kernel on the gathered cache, bit for bit."""
    lib, code, st = load(), DTYPE_CODE[dtype], stream_ptr(DEV)
    L = 8192 if kind == "batch" else 131072
    pos = [L - 1, 0, 4097, 64] if kind == "batch" else [L - 1, 0, 70001, 8192]
    B = len(pos)
    tab, N = table([p + 1 for p in pos], L // PG, hq + hkv)
    cos, sin = R.tables(L, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq + hkv)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV).to(dtype)
    q, k, v = rn(B, hq * R.HD), rn(B, hkv * R.HD), rn(B, hkv * R.HD)
    if kind == "kv8":
        names = ("kq", "ks", "kz", "vq", "vs", "vz")
        pool = {n: torch.randint(0, 256, (N + 1, hkv, PG, R.HD), generator=gen, device=DEV, dtype=torch.uint8) for n in ("kq", "vq")}
        for n in ("ks", "vs"):
            pool[n] = (torch.rand(N + 1, hkv, PG, 2, generator=gen, device=DEV) * 0.02 + 0.005).to(dtype)
        for n in ("kz", "vz"):
            pool[n] = (torch.rand(N + 1, hkv, PG, 2, generator=gen, device=DEV) * 255).to(dtype)
    else:
        names = ("kc", "vc")
        pool = {"kc": rn(N + 1, hkv, PG, R.HD), "vc": rn(N + 1, hkv, PG, R.HD)}
    flat = {n: gather(t, tab) for n, t in pool.items()}
    p = torch.tensor(pos, dtype=torch.int64, device=DEV)
    outs, wss = [], []
    for paged, c in ((True, pool), (False, flat)):
        out = torch.zeros(B, hq * R.HD, dtype=dtype, device=DEV)
        ws = torch.zeros(lib.hqq_b200_glue_rope_attn_decode_split_workspace_bytes(hq, hkv, R.HD, B), dtype=torch.uint8, device=DEV)
        head = [ptr(q), ptr(k), ptr(v), ptr(cos), ptr(sin)] + [ptr(c[n]) for n in names]
        sfx = "_paged" if paged else "_seqpos"
        mid = ([ptr(tab)] if paged else []) + [ptr(p), ptr(out)]
        tail = [hq, hkv, L, R.HD] + ([64] if kind == "kv8" else []) + [B] + ([N] if paged else []) + [code, st]
        if kind == "batch":
            check(getattr(lib, "hqq_b200_glue_rope_attn_decode_batch" + sfx)(*head, *mid, *tail))
        elif kind == "split":
            check(getattr(lib, "hqq_b200_glue_rope_attn_decode_split" + sfx)(*head, *mid, ptr(ws), *tail))
        else:
            check(getattr(lib, "hqq_b200_glue_rope_attn_decode_split_kv8" + sfx)(*head, *mid, ptr(ws), *tail))
        outs.append(out)
        wss.append(ws)
    torch.cuda.synchronize(DEV)
    assert torch.equal(outs[0], outs[1])
    assert torch.count_nonzero(wss[0][-4 * B * hkv:]) == 0
    for n in names:
        g = gather(pool[n], tab)
        for b, x in enumerate(pos):
            assert torch.equal(g[b, :, :x + 1], flat[n][b, :, :x + 1]), (n, b)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", HEADS)
def test_paged_prefill_equals_varlen_on_gathered_cache(hq, hkv, dtype):
    """n_tok [1000, 0, 333, 1] at pos0 [0, 5, 131072 - 333, 131071]: rows kernel and attention equal the _varlen kernels on the
    gathered cache, bit for bit."""
    lib, code, st = load(), DTYPE_CODE[dtype], stream_ptr(DEV)
    L, n_tok, pos0 = 131072, [1000, 0, 333, 1], [0, 5, 131072 - 333, 131071]
    B, M = len(n_tok), sum(n_tok)
    tab, N = table([p + n if n else p for p, n in zip(pos0, n_tok)], L // PG, 3 * hq + hkv)
    cos, sin = R.tables(L, dtype, DEV)
    gen = torch.Generator(device=DEV).manual_seed(hq * 3 + hkv)
    rn = lambda *s: torch.randn(*s, generator=gen, device=DEV).to(dtype)
    q, k, v = rn(M, hq * R.HD), rn(M, hkv * R.HD), rn(M, hkv * R.HD)
    kp, vp = rn(N + 1, hkv, PG, R.HD), rn(N + 1, hkv, PG, R.HD)
    kc, vc = gather(kp, tab), gather(vp, tab)
    qo, qo2, out, out2 = (torch.zeros_like(q) for _ in range(4))
    check(lib.hqq_b200_glue_rope_append_rows_paged(ptr(q), ptr(k), ptr(v), ptr(cos), ptr(sin), ptr(kp), ptr(vp), ptr(tab), ptr(qo), ints(pos0), ints(n_tok),
                                                   hq, hkv, L, R.HD, B, N, code, st))
    check(lib.hqq_b200_glue_attn_prefill_paged(ptr(qo), ptr(kp), ptr(vp), ptr(tab), ptr(out), ints(pos0), ints(n_tok), hq, hkv, L, R.HD, B, N, code, st))
    check(lib.hqq_b200_glue_rope_append_rows_varlen(ptr(q), ptr(k), ptr(v), ptr(cos), ptr(sin), ptr(kc), ptr(vc), ptr(qo2), ints(pos0), ints(n_tok), hq,
                                                    hkv, L, R.HD, B, code, st))
    check(lib.hqq_b200_glue_attn_prefill_varlen(ptr(qo2), ptr(kc), ptr(vc), ptr(out2), ints(pos0), ints(n_tok), hq, hkv, L, R.HD, B, code, st))
    torch.cuda.synchronize(DEV)
    assert torch.equal(qo, qo2) and torch.equal(out, out2)
    for b in range(B):
        e = pos0[b] + n_tok[b]
        assert torch.equal(gather(kp, tab)[b, :, :e], kc[b, :, :e]) and torch.equal(gather(vp, tab)[b, :, :e], vc[b, :, :e]), b


# ------------------------------------------------------------------------------------------------ DecodeModel(kv_pages=N)
SHAPE = harness.LLAMA3_8B
_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    """The models (and their captured graphs) live for this module only: the suite runs in one process."""
    yield
    _MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _model(dtype, kv_pages, kv_bits=16, cache_len=2048, fused=True, **kw):
    key = (dtype, kv_pages, kv_bits, cache_len, fused, tuple(sorted(kw.items())))
    if key not in _MODELS:
        m = harness.DecodeModel(SHAPE, n_layers=2, dtype=dtype, device=DEV, cache_len=cache_len, fused=fused, seed=11, batch=4, ragged=True,
                                kv_bits=kv_bits, kv_pages=kv_pages, **kw)
        m.capture()
        _MODELS[key] = m
    return _MODELS[key]


def _pair(dtype, kv_bits=16, cache_len=2048, fused=True, kv_pages=None, **kw):
    """The unpaged ragged model and its paged twin (by default with as many pages as the contiguous caches hold)."""
    return (_model(dtype, None, kv_bits, cache_len, fused, **kw),
            _model(dtype, kv_pages or 4 * cache_len // PG, kv_bits, cache_len, fused, **kw))


def _caches(m, b, end):
    out = []
    for blk in m.blocks:
        cv = m.cache_view(blk)
        out += [cv[n][b, :, :end].clone() for n in harness.DecodeModel._CACHE_NAMES if n in cv]
    return out


def _steps(m, n):
    toks, logits = [], []
    for _ in range(n):
        m.decode()
        toks.append(m.next_tok.clone())
        if m.fused:
            logits.append(m._bufs["logits"].clone())
    torch.cuda.synchronize(DEV)
    return toks, logits


def _prompts(lengths, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, SHAPE.vocab, (n,), generator=g, device=DEV) for n in lengths]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _copy_slot(m, src, dst):
    """The unpaged counterpart of fork: slot src's caches, position and token copied into slot dst."""
    for blk in m.blocks:
        for n in harness.DecodeModel._CACHE_NAMES:
            if n in blk:
                blk[n][dst].copy_(blk[n][src])
    m.pos[dst].copy_(m.pos[src])
    m.tok[dst].copy_(m.tok[src])


@pytest.mark.parametrize("kv_bits,cache_len", [(16, 2048), (16, 16384), (8, 2048), (8, 16384)], ids=["single", "split", "kv8", "kv8_16k"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_paged_model_equals_unpaged(dtype, kv_bits, cache_len):
    """Packed prefill of 1, 37, 300 and 1000 tokens, 70 decode() steps across page edges, a refill of slot 2, 20 more steps: tokens,
    last_logits, step logits and the gathered caches equal the unpaged ragged model's bit for bit."""
    prompts, refill = _prompts([1, 37, 300, 1000], 3), _prompts([23], 4)[0]
    runs = []
    for m in _pair(dtype, kv_bits, cache_len):
        m.reset_state()
        t0 = m.prefill(prompts, chunk=256)
        l0 = m.last_logits.clone()
        a = _steps(m, 70)
        t1 = m.prefill([None, None, refill, None], chunk=16)
        l1 = m.last_logits.clone()
        c = _steps(m, 20)
        assert m.pos.tolist() == [91, 127, 43, 1090]
        runs.append((t0, l0, a, t1, l1, c, [_caches(m, b, e) for b, e in enumerate(m.pos.tolist())]))
    (t0, l0, a, t1, l1, c, ca), (u0, k0, x, u1, k1, y, cb) = runs
    assert torch.equal(t0, u0) and torch.equal(l0, k0) and torch.equal(t1, u1) and torch.equal(l1, k1)
    assert _same(a[0], x[0]) and _same(a[1], x[1]) and _same(c[0], y[0]) and _same(c[1], y[1])
    for p, q in zip(ca, cb):
        assert _same(p, q)


@pytest.mark.parametrize("kv_bits", [16, 8])
def test_paged_release_leaves_other_slots_alone(kv_bits):
    """release(1) after 10 steps: slots 0, 2 and 3 keep the tokens and logits of a run without it bit for bit, and free_pages rises
    by the slot's pages."""
    prompts = _prompts([5, 140, 17, 100], 5)
    _, m = _pair(torch.float16, kv_bits)
    runs = []
    for rel in (False, True):
        m.reset_state()
        m.prefill(prompts, chunk=64)
        t1, g1 = _steps(m, 10)
        if rel:
            held, free = m.pages.pages_of(1), m.free_pages
            assert held == 3
            m.release(1)
            assert m.free_pages == free + held
            assert int((m.page_table[1] != m.kv_pages).sum()) == 0
        t2, g2 = _steps(m, 70)
        runs.append((torch.stack(t1 + t2), torch.stack(g1 + g2)))
    keep = [0, 2, 3]
    assert torch.equal(runs[0][0][:, keep], runs[1][0][:, keep]) and torch.equal(runs[0][1][:, keep], runs[1][1][:, keep])


@pytest.mark.parametrize("do_sample", [False, True], ids=["greedy", "sample"])
def test_paged_fork(do_sample):
    """A 300-token prompt in slot 0 forked to slots 1-3: 5 + 3 pages in use; the streams equal the unpaged model with slot 0's cache
    copied into slots 1-3, bit for bit (greedy: four identical streams; do_sample: four different ones).  Then a different suffix per
    slot at start = pos: equal again."""
    kw = {"do_sample": True, "top_k": 50, "temperature": 1.0} if do_sample else {}
    prompt = _prompts([300], 6)[0]
    suffixes = _prompts([5, 64, 100, 1], 7)
    u, m = _pair(torch.float16, **kw)
    runs = []
    for x in (m, u):
        x.reset_state()
        x.prefill([prompt, None, None, None])
        for d in (1, 2, 3):
            if x is m:
                x.fork(0, d)
            else:
                _copy_slot(x, 0, d)
        if x is m:
            assert m.kv_pages - m.free_pages == 8
        s1 = _steps(x, 30)
        x.reset_state()
        x.prefill([prompt, None, None, None])
        for d in (1, 2, 3):
            x.fork(0, d) if x is m else _copy_slot(x, 0, d)
        t = x.prefill(suffixes, start=300, chunk=32)
        lg = x.last_logits.clone()
        s2 = _steps(x, 30)
        runs.append((s1, t, lg, s2, [_caches(x, b, e) for b, e in enumerate(x.pos.tolist())]))
    (a1, ta, la, a2, ca), (b1, tb, lb, b2, cb) = runs
    assert _same(a1[0], b1[0]) and _same(a1[1], b1[1]) and torch.equal(ta, tb) and torch.equal(la, lb)
    assert _same(a2[0], b2[0]) and _same(a2[1], b2[1])
    for p, q in zip(ca, cb):
        assert _same(p, q)
    streams = torch.stack(a1[0])  # [steps, 4]
    same = all(torch.equal(streams[:, 0], streams[:, d]) for d in (1, 2, 3))
    assert same != do_sample


def test_paged_wrap_equals_unpaged():
    """cache_len 256: slots wrap past the end of the cache and stay equal to the unpaged model."""
    prompts = _prompts([200, 5, 255, 64], 8)
    runs = []
    for m in _pair(torch.float16, cache_len=256):
        m.reset_state()
        t = m.prefill(prompts)
        runs.append((t, _steps(m, 150)))
    assert torch.equal(runs[0][0], runs[1][0]) and _same(runs[0][1][0], runs[1][1][0]) and _same(runs[0][1][1], runs[1][1][1])


def test_paged_out_of_pages_changes_nothing():
    """An undersized pool: a prefill that needs more pages than are free raises RuntimeError and leaves the allocator, the device
    table and the positions as they were."""
    m = _model(torch.float16, 12)
    m.reset_state()
    m.prefill(_prompts([300, 100, 10, 10], 9))  # 5 + 2 + 1 + 1 pages
    before = ([r[:] for r in m.pages.table], m.pages.ref[:], sorted(m.pages.free), m.page_table.clone(), m.pos.clone())
    with pytest.raises(RuntimeError):
        m.prefill([None, None, _prompts([400], 10)[0], None])
    after = ([r[:] for r in m.pages.table], m.pages.ref[:], sorted(m.pages.free), m.page_table.clone(), m.pos.clone())
    assert before[:3] == after[:3] and torch.equal(before[3], after[3]) and torch.equal(before[4], after[4])


def test_paged_reference_equals_unpaged_reference():
    """fused=False: the paged reference walk (framework indexing through the table, then SDPA) equals the unpaged one bit for bit
    through the prefill (tokens, last_logits, caches).  Its decode steps are not run-to-run deterministic even unpaged (two identical
    unpaged runs differ by an ulp in a few layer-1 rows on the H100), so there the tokens must agree and the caches stay within 1e-3."""
    prompts, refill = _prompts([1, 37, 70, 130], 11), _prompts([9], 12)[0]
    runs = []
    for m in _pair(torch.float16, fused=False):
        m.reset_state()
        t0 = m.prefill(prompts, chunk=64)
        l0 = m.last_logits.clone()
        c0 = [_caches(m, b, e) for b, e in enumerate(m.pos.tolist())]
        a = _steps(m, 10)
        t1 = m.prefill([None, refill, None, None])
        c = _steps(m, 5)
        runs.append((t0, l0, c0, a[0], t1, c[0], [_caches(m, b, e) for b, e in enumerate(m.pos.tolist())]))
    (t0, l0, c0, a, t1, c, ca), (u0, k0, d0, x, u1, y, cb) = runs
    assert torch.equal(t0, u0) and torch.equal(l0, k0)
    for p, q in zip(c0, d0):
        assert _same(p, q)
    assert torch.equal(t1, u1) and _same(a, x) and _same(c, y)
    for p, q in zip(ca, cb):
        for u, w in zip(p, q):
            assert float((u.float() - w.float()).norm() / w.float().norm().clamp_min(1e-30)) <= 1e-3


def test_paged_options_rejected():
    for kw in ({"ragged": False, "kv_pages": 8}, {"ragged": True, "kv_pages": 0}, {"ragged": True, "kv_pages": 8, "cache_len": 100}):
        with pytest.raises(ValueError):
            harness.DecodeModel(harness.TINY, n_layers=1, device=DEV, **{"cache_len": 256, **kw})
