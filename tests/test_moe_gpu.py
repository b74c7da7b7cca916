"""GPU: the mixture-of-experts path -- the router, the expert-grouped small-M kernel and the combine at Mixtral sizes against
tests/moe_ref.py and the float64 bound of tests/fused_ref.py, and the decode harness's MoE blocks (fused against fused=False, paged
against unpaged, speculative, quantised caches, per-slot sampling, the MIXTRAL_8X7B shape)."""
import pytest
import torch

import fused_ref as FR
import moe_ref as MR
from hqq_b200 import harness, ops
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SMALL = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048, n_experts=8, experts_per_token=2)


def route(x, router, k):
    lib = load()
    M, H = x.shape
    E = router.shape[0]
    i32 = lambda *s: torch.full(s, -1, dtype=torch.int32, device=DEV)
    out = {"ids": i32(M, k), "w": torch.zeros(M, k, device=DEV), "pair_of": i32(M, k), "off": i32(E), "cnt": i32(E), "token": i32(M * k)}
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    check(lib.hqq_b200_glue_moe_route(ptr(x), ptr(router), M, H, E, k, ptr(out["ids"]), ptr(out["w"]), ptr(out["pair_of"]), ptr(out["off"]),
                                      ptr(out["cnt"]), ptr(out["token"]), ptr(ticket), DTYPE_CODE[x.dtype], stream_ptr(DEV)))
    torch.cuda.synchronize()
    assert int(ticket) == 0
    return out


@pytest.mark.parametrize("M", [1, 32, 256, 4096])
def test_router_at_mixtral_size(M):
    g = torch.Generator(device=DEV).manual_seed(M)
    H, E, k = 4096, 8, 2
    x = torch.randn(M, H, device=DEV, generator=g).half()
    router = (torch.randn(E, H, device=DEV, generator=g) * 0.02).half()
    out = route(x, router, k)
    ids, w, p = MR.route(x, router, k)
    keep = ~MR.near_tie(p, k)
    assert torch.equal(out["ids"][keep], ids[keep]) and int((~keep).sum()) <= max(1, M // 50)
    # the kernel rounds an fp32 sum to fp16, the restatement the exact one: a logit next to a rounding boundary may land one fp16 ulp
    # (2^-11 relative) away, which moves that row's weights by about as much; every other row matches to fp32 rounding
    err = ((out["w"] - w).abs() / w).max(dim=1).values[keep]
    assert float(err.max()) <= 2e-3 and int((err > 2e-6).sum()) <= max(1, M // 100), (float(err.max()), int((err > 2e-6).sum()))
    off, cnt, token, pair_of = MR.group(out["ids"].cpu(), E)
    assert torch.equal(out["off"].cpu(), off) and torch.equal(out["cnt"].cpu(), cnt)
    assert torch.equal(out["token"].cpu(), token) and torch.equal(out["pair_of"].cpu(), pair_of)


def _experts(E, N, K, seed, nbits=4, gs=64, dtype=torch.float16):
    g = FR.generator(seed, DEV)
    layers = [FR.draw_layer(g, N, K, nbits, gs, dtype, pack=ops.pack) for _ in range(E)]
    st = lambda f: torch.stack([f(L) for L in layers]).contiguous()
    return layers, (st(lambda L: L.W_q), st(lambda L: L.s.reshape(-1)), st(lambda L: L.z.reshape(-1)))


def _ids(M, E, k, skew, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.rand(M, E, device=DEV, generator=g)
    if skew:
        s[: M * 7 // 8, 0] += 2.0  # most rows go to expert 0
    return torch.topk(s, k, dim=-1).indices.to(torch.int32)


@pytest.mark.parametrize("skew", [False, True], ids=["even", "skewed"])
@pytest.mark.parametrize("M", [1, 32, 256, 4096])
def test_grouped_gate_up_and_down_at_mixtral_size(M, skew):
    """Grouped gate/up (rows gathered by token) and grouped down (rows in pair order) against float64 per expert; a sample of experts
    at M = 4096 keeps the float64 work small.  The scale of every expert the routing did not select is NaN: unselected experts are
    never read, so the outputs stay finite."""
    E, k, H, I = 8, 2, 4096, 14336
    ids = _ids(M, E, k, skew, M)
    if M == 1:
        ids = torch.tensor([[2, 6]], dtype=torch.int32, device=DEV)
    off, cnt, token, _ = (t.to(DEV) for t in MR.group(ids.cpu(), E))
    used = set(ids.view(-1).tolist())
    gl, gs_ = _experts(E, I, H, 1)
    ul, us_ = _experts(E, I, H, 2)
    dl, ds_ = _experts(E, H, I, 3)
    for stk in (gs_, us_, ds_):
        for e in range(E):
            if e not in used:
                stk[1][e].fill_(float("nan"))
    x = FR.draw_x(FR.generator(4, DEV), M, H, 64, torch.float16)
    P_ = M * k
    gate = torch.empty(P_, I, device=DEV, dtype=torch.float16)
    up = torch.empty_like(gate)
    ops.linear_fwd_grouped(x, token, (gs_, us_), [gate, up], off, cnt, P_, 64, 4)
    act = FR.draw_x(FR.generator(5, DEV), P_, I, 64, torch.float16)  # the down projection's rows, in pair order
    down = torch.empty(P_, H, device=DEV, dtype=torch.float16)
    ops.linear_fwd_grouped(act, None, (ds_,), [down], off, cnt, P_, 64, 4)
    torch.cuda.synchronize()
    for t in (gate, up, down):
        assert bool(torch.isfinite(t).all())
    experts = [e for e in range(E) if int(cnt[e])]
    for e in experts if M < 4096 else experts[:2]:
        a, c = int(off[e]), min(int(cnt[e]), 64)
        rows = x[token[a:a + c].long()]
        FR.check(gate[a:a + c], FR.reference(gl[e], rows, 1), f"gate {e}")
        FR.check(up[a:a + c], FR.reference(ul[e], rows, 1), f"up {e}")
        FR.check(down[a:a + c], FR.reference(dl[e], act[a:a + c], 1), f"down {e}")
    # bit-identical with finite scales on the unselected experts
    for stk in (gs_, us_):
        for e in range(E):
            if e not in used:
                stk[1][e].fill_(0.01)
    gate2, up2 = torch.empty_like(gate), torch.empty_like(up)
    ops.linear_fwd_grouped(x, token, (gs_, us_), [gate2, up2], off, cnt, P_, 64, 4)
    assert torch.equal(gate2, gate) and torch.equal(up2, up)


@pytest.mark.parametrize("k", [1, 2, 4])
def test_combine_bit_exact_at_mixtral_size(k):
    M, E, H = 64, 8, 4096
    ids = _ids(M, E, k, False, 7)
    g = torch.Generator(device=DEV).manual_seed(k)
    w = torch.softmax(torch.randn(M, k, device=DEV, generator=g), dim=-1)
    _, _, _, pair_of = MR.group(ids.cpu(), E)
    pair_of = pair_of.to(DEV)
    y = torch.randn(M * k, H, device=DEV, generator=g).half()
    delta = torch.empty(M, H, device=DEV, dtype=torch.float16)
    check(load().hqq_b200_glue_moe_combine(ptr(y), ptr(ids), ptr(w), ptr(pair_of), ptr(delta), M, H, k, DTYPE_CODE[torch.float16], stream_ptr(DEV)))
    assert torch.equal(delta, MR.combine(y, ids, w, pair_of, E))


# ---- harness ---------------------------------------------------------------------------------------------------------------------
def _model(fused=True, batch=1, ragged=False, shape=SMALL, **kw):
    return harness.DecodeModel(shape, dtype=torch.float16, device=DEV, cache_len=kw.pop("cache_len", 512), fused=fused, seed=3, batch=batch,
                               ragged=ragged, **kw)


def _decode(m, n):
    toks, logits = [], []
    for _ in range(n):
        m.decode()
        toks.append(m.next_tok.clone())
        if m.fused:
            logits.append(m._bufs["logits"].clone())
    torch.cuda.synchronize()
    return torch.stack(toks), logits


def _prompts(lengths, seed, vocab=SMALL.vocab):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, vocab, (n,), generator=g, device=DEV) for n in lengths]


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("batch", [1, 4])
def test_moe_model_fused_matches_framework_ops(batch):
    """Prefill (ragged batch of 4: prompts of 5, 37, 100 and 300 tokens) and 16 captured decode steps: prefill logits within the
    prefill bar, and the greedy tokens equal -- the early ones exactly, later ones up to fp16 near-ties."""
    runs = []
    for fused in (True, False):
        m = _model(fused, batch=batch, ragged=batch > 1)
        assert m.fused is fused and m.quantized_weights > 8 * 3 * 2048 * 1024
        m.capture()
        m.reset_state()
        prompts = _prompts([5, 37, 100, 300][:batch], 1)
        tok = m.prefill(prompts if batch > 1 else prompts[0].view(1, -1), chunk=128)
        runs.append((tok.view(-1), m.last_logits.clone(), _decode(m, 16)[0]))
        del m
    (_, la, sa), (_, lb, sb) = runs
    assert _rel(la, lb) <= 2e-3, _rel(la, lb)
    assert torch.equal(sa[:2], sb[:2]), (sa[:2], sb[:2])
    assert (sa == sb).float().mean().item() >= 0.85, (sa, sb)


def test_moe_paged_equals_unpaged():
    prompts = _prompts([1, 37, 300, 100], 3)
    runs = []
    for pages in (None, 64):
        m = _model(True, batch=4, ragged=True, kv_pages=pages)
        m.capture()
        m.reset_state()
        t0 = m.prefill(prompts, chunk=128)
        toks, logits = _decode(m, 70)
        runs.append((t0, m.last_logits.clone(), toks, logits))
    (a0, al, at, ag), (b0, bl, bt, bg) = runs
    assert torch.equal(a0, b0) and torch.equal(al, bl) and torch.equal(at, bt)
    assert all(torch.equal(x, y) for x, y in zip(ag, bg))


def test_moe_spec_follows_decode_and_verify_meets_reference():
    K = 3
    prompts = _prompts([40, 80, 120, 160], 10)
    m = _model(True, batch=4, ragged=True, spec_k=K)
    m.capture()
    m.capture_spec()
    m.reset_state()
    m.prefill(prompts, chunk=256)
    saved = (m.pos.clone(), m.tok.clone(), m.hist.clone(), [{n: blk[n].clone() for n in ("k_cache", "v_cache")} for blk in m.blocks])
    plain = []
    for _ in range(24):
        plain.append(m.tok.clone())
        m.decode()
    plain = torch.stack(plain, 1)
    pos, tok, hist, caches = saved
    m.pos.copy_(pos); m.tok.copy_(tok); m.hist.copy_(hist)
    for blk, c in zip(m.blocks, caches):
        for n, t in c.items():
            blk[n].copy_(t)
    spec = [[int(m.tok[b])] for b in range(4)]
    while min(len(s) for s in spec) < 24:
        toks, n_new = m.decode_spec()
        for b in range(4):
            spec[b] += toks[b, :int(n_new[b])].tolist()
    # The verify pass rounds differently (M = batch (K + 1) rows).  In a dense model that can only flip a near tie of the logits; here a
    # last-bit difference in a router logit can also select another expert for one row, after which the two streams are different
    # valid continuations.  So: the first tokens of every slot agree, and most of the run agrees before any stream leaves decode()'s.
    first = []
    for b in range(4):
        got = torch.tensor(spec[b][:24], device=DEV)
        assert got[:2].tolist() == plain[b, :2].tolist(), b
        miss = (got != plain[b]).nonzero().view(-1).tolist()
        first.append(miss[0] if miss else 24)
    assert sum(first) >= 0.6 * 4 * 24, first
    # the fused verify against verify() from one state
    g = torch.Generator(device=DEV).manual_seed(9)
    d = torch.randint(0, 50, (4, K), device=DEV, generator=g)
    tok = torch.randint(0, 50, (4,), device=DEV, generator=g)
    r = _model(False, batch=4, ragged=True, spec_k=K)
    r.reset_state()
    out = []
    for x in (m, r):
        x.pos.copy_(pos)
        for bx, c in zip(x.blocks, caches):
            for n, t in c.items():
                bx[n].copy_(t)
        x.tok.copy_(tok)
        x._spec_drafts.copy_(d)
        with torch.no_grad():
            (x.spec_graph.replay if x.fused else x.verify)()
        out.append(x.spec_logits.float().clone())
    assert _rel(out[0], out[1]) <= 2e-3, _rel(out[0], out[1])


@pytest.mark.parametrize("kw", [{"kv_bits": 8}, {"kv_bits": 4, "kv_group_size": 64}, {"slot_sampling": True}], ids=["kv8", "kv4", "slots"])
def test_moe_options_capture_and_are_deterministic(kw):
    runs = []
    for _ in range(2):
        m = _model(True, batch=4, ragged=True, **kw)
        if kw.get("slot_sampling"):
            m.set_sampling(1, temperature=0.8, top_k=20)
            m.set_sampling(2, repetition_penalty=1.3)
        m.capture()
        m.reset_state()
        m.prefill(_prompts([5, 37, 100, 300], 2), chunk=128)
        toks, logits = _decode(m, 12)
        assert all(bool(torch.isfinite(l).all()) for l in logits)
        runs.append((toks, logits))
        del m
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


@pytest.mark.parametrize("batch", [1, 32])
def test_mixtral_8x7b_two_layers(batch):
    runs = []
    for fused in (True, False):
        m = _model(fused, batch=batch, ragged=batch > 1, shape=harness.MIXTRAL_8X7B, n_layers=2, cache_len=256)
        m.capture()
        m.reset_state()
        m.tok.copy_(torch.arange(3, 3 + batch, device=DEV))
        runs.append(_decode(m, 8)[0])
        del m
        torch.cuda.empty_cache()
    a, b = runs
    assert torch.equal(a[:2], b[:2]), (a[:2], b[:2])


def test_dense_step_launch_count_is_unchanged():
    """A dense block's captured step issues 8 launches, a mixture-of-experts block 10 (route, grouped gate/up, SiLU*mul, grouped
    down and combine in place of gate/up, SiLU*mul and down); what surrounds the blocks does not change."""
    lib = load()

    def launches(n_experts, n_layers, batch):
        shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=n_layers, n_heads=8, n_kv_heads=2, vocab=2048, n_experts=n_experts)
        m = harness.DecodeModel(shape, dtype=torch.float16, device=DEV, cache_len=64, fused=True, seed=3, batch=batch)
        m.capture()
        torch.cuda.synchronize()
        lib.hqq_b200_launch_count_reset()
        m.step_fused()
        torch.cuda.synchronize()
        return int(lib.hqq_b200_launch_count())
    for batch in (1, 4):
        base = launches(0, 0, batch)
        assert launches(0, 2, batch) - base == 2 * 8, batch
        assert launches(8, 2, batch) - base == 2 * 10, batch
