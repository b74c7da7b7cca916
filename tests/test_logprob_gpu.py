"""Prompt scoring on the H100: the LSE head (hqq_b200_lm_logprob) at the Llama vocabularies, and DecodeModel.score() on a 2-layer
Llama-3-8B-shaped model.

Kernel: lse and tgt within logprob_ref's bound of float64 log-softmax over the T-rounded float64 logits at vocabulary 128256, 16032
(the tp = 8 shard, a ragged last tile) and 32000, M up to 4096; a position's values do not depend on the rows around it.
Harness: score() leaves the state prefill() leaves bit for bit (ragged prompts of 1, 37, 300 and 1000 tokens; kv_bits 8; kv_pages;
do_sample; spec_k), its log-probabilities meet the prefill tests' bars against the fused=False reference, and their chunk
dependence is the prefill walk's own: the LSE head is row-invariant, so only the residual stream it is fed changes with the chunk.
tools/perplexity.py gives the fused=False windows' perplexity."""
import math
import os
import sys

import pytest
import torch

import logprob_ref as R
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import perplexity  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TOL = {torch.float16: 2e-3, torch.bfloat16: 1e-2}  # the prefill tests' relative L2 bars (DESIGN §3.5)


def lm_logprob(x, W, targets, index_offset=0):
    lib = load()
    M, K = x.shape
    N = W.shape[0]
    ws = torch.empty(lib.hqq_b200_lm_logprob_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
    lse = torch.full((M,), float("nan"), device=DEV)
    tgt = torch.full((M,), float("nan"), device=DEV)
    check(lib.hqq_b200_lm_logprob(ptr(x), ptr(W), ptr(targets), ptr(lse), ptr(tgt), ptr(ws), M, N, K, index_offset, DTYPE_CODE[x.dtype],
                                  stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return lse, tgt


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("N", [128256, 16032, 32000])
def test_lse_head_within_the_float64_bound(dtype, N):
    K = 4096
    g = torch.Generator(device=DEV).manual_seed(N)
    off = 7 * N if N == 16032 else 0  # the tp = 8 shard of rank 7
    x = torch.randn(4096, K, generator=g, device=DEV).to(dtype)
    W = (torch.randn(N, K, generator=g, device=DEV) * (2.0 / math.sqrt(K))).to(dtype)
    t = torch.randint(off, off + N, (4096,), generator=g, device=DEV)
    t[:6] = torch.tensor([-1, off, off + N - 1, off - 1, off + N, 10 ** 9])
    lse, tgt = lm_logprob(x, W, t, off)
    for r0 in range(0, 4096, 256):  # float64 reference in row blocks
        sl = slice(r0, r0 + 256)
        ref_lse, ref_tgt, L, absdot = R.reference(x[sl], W, t[sl], off)
        b_lse, b_tgt = R.bounds(x[sl], W, t[sl], off, L, absdot, ref_lse)
        assert bool(((lse[sl].double() - ref_lse).abs() <= b_lse).all()), r0
        out = ref_tgt.isinf()
        assert bool((tgt[sl][out] == -math.inf).all())
        assert bool(((tgt[sl].double()[~out] - ref_tgt[~out]).abs() <= b_tgt[~out]).all()), r0
        del L, absdot
    for M, at in ((1, 0), (300, 0), (17, 4000)):  # the same rows inside other blocks: identical bits
        l2, t2 = lm_logprob(x[at:at + M].contiguous(), W, t[at:at + M].contiguous(), off)
        assert torch.equal(l2, lse[at:at + M]) and torch.equal(t2, tgt[at:at + M]), (M, at)


# ------------------------------------------------------------------------------------------------ DecodeModel.score()
SHAPE = harness.LLAMA3_8B
LENGTHS = (1, 37, 300, 1000)
_MODELS = {}


def _model(dtype, fused=True, **kw):
    key = (dtype, fused, tuple(sorted(kw.items())))
    if key not in _MODELS:
        _MODELS.clear()
        torch.cuda.empty_cache()
        _MODELS[key] = harness.DecodeModel(SHAPE, n_layers=2, dtype=dtype, device=DEV, cache_len=2048, fused=fused, seed=11, batch=4,
                                           ragged=True, **kw)
    return _MODELS[key]


def _prompts(seed=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randint(0, SHAPE.vocab, (n,), generator=g, device=DEV) for n in LENGTHS]


def _state(m):
    st = {"tok": m.tok.clone(), "pos": m.pos.clone(), "last_logits": m.last_logits.clone(), "ctr": m._sample_ctr.clone()}
    for i, blk in enumerate(m.blocks):
        for n in m._CACHE_NAMES:
            if n in blk:
                st[f"{i}.{n}"] = blk[n].clone()
    if m.kv_pages is not None:
        st["table"] = m.page_table.clone()
        st["free"] = m.free_pages
    if m.spec_k is not None:
        st["hist"] = m.hist.clone()
    return st


@pytest.mark.parametrize("cfg", [{}, {"kv_bits": 8}, {"kv_pages": 80}, {"do_sample": True}, {"spec_k": 3}],
                         ids=["kv16", "kv8", "paged", "sample", "spec"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_score_leaves_the_state_prefill_leaves(dtype, cfg):
    m = _model(dtype, **cfg)
    prompts = _prompts()
    m.reset_state()
    tok = m.prefill(prompts, chunk=256)
    want = _state(m)
    m.reset_state()
    lps = m.score(prompts, chunk=256)
    torch.cuda.synchronize(DEV)
    got = _state(m)
    assert torch.equal(tok, m.tok)
    for k in want:
        assert (want[k] == got[k]) if not torch.is_tensor(want[k]) else torch.equal(want[k], got[k]), k
    assert [lp.numel() for lp in lps] == [n - 1 for n in LENGTHS]
    assert all(bool(torch.isfinite(lp).all()) and bool((lp <= 0).all()) for lp in lps)


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("kv_bits", [16, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_score_matches_the_reference_and_chunking(dtype, kv_bits):
    """The fused log-probabilities against fused=False (torch.matmul logits, fp32 log_softmax, gather) within the prefill bars, per
    slot; chunk 2048 against chunk 256: the LSE head is bit for bit row-invariant (test above), so the two differ only as the
    prefill walk's residual stream does with the chunk -- held to the same bar, as the prefill's own last_logits are."""
    tol = TOL[dtype] * (2.5 if kv_bits == 8 and dtype == torch.float16 else 1)  # kv8 fp16: tests/test_ragged_gpu.py's 5e-3
    prompts = _prompts(5)
    m = _model(dtype, kv_bits=kv_bits)
    res = {}
    for chunk in (256, 2048):
        m.reset_state()
        res[chunk] = ([lp.clone() for lp in m.score(prompts, chunk=chunk)], m.last_logits.clone())
    r = _model(dtype, fused=False, kv_bits=kv_bits)
    r.reset_state()
    ref = r.score(prompts, chunk=256)
    for b, n in enumerate(LENGTHS):
        if n == 1:
            assert res[256][0][b].numel() == 0 and ref[b].numel() == 0
            continue
        assert _rel(res[256][0][b], ref[b]) <= tol, (b, _rel(res[256][0][b], ref[b]))
        assert _rel(res[2048][0][b], res[256][0][b]) <= tol, b
    assert _rel(res[2048][1], res[256][1]) <= tol


def test_lock_step_score_matches_ragged():
    """Lock-step score() ([batch, T - 1]) against the ragged model on equal-length prompts: the same bits."""
    prompt = torch.randint(0, SHAPE.vocab, (4, 300), generator=torch.Generator(device=DEV).manual_seed(8), device=DEV)
    m = harness.DecodeModel(SHAPE, n_layers=2, dtype=torch.float16, device=DEV, cache_len=2048, seed=11, batch=4, ragged=False)
    a = m.score(prompt, chunk=128)
    del m
    torch.cuda.empty_cache()
    b = _model(torch.float16).score(list(prompt.unbind(0)), chunk=128)
    assert a.shape == (4, 299)
    assert all(torch.equal(a[i], b[i]) for i in range(4))


def test_perplexity_tool_equals_the_reference_windows():
    """tools/perplexity.py's windows over a short random stream, fused against fused=False: per-window log-probabilities within the
    fp16 bar and the same perplexity to that accuracy."""
    g = torch.Generator().manual_seed(0)
    tokens = torch.randint(0, 32000, (1500,), generator=g).to(DEV)
    wins = perplexity.windows(tokens.numel(), 512, 256)
    out = {}
    for fused in (True, False):
        m = _model(torch.float16, fused=fused)
        m.reset_state()
        out[fused] = perplexity.score_windows(m, tokens, wins, 4)
    for a, b in zip(out[True], out[False]):
        assert _rel(a, b) <= TOL[torch.float16]
    p, q = perplexity.perplexity(wins, out[True]), perplexity.perplexity(wins, out[False])
    assert abs(math.log(p) - math.log(q)) <= TOL[torch.float16] * abs(math.log(q))
