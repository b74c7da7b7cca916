"""The LSE head (csrc/linear_gemm.cu: the dense wgmma kernel's LSE epilogue and the tile merge, hqq_b200_lm_logprob) on the CPU kernel
emulator, held to float64 log-softmax of the T-rounded float64 logits within logprob_ref's bound; row invariance bit for bit; four
planted defects that must each leave the bound; argument checks; and the perplexity tool's window arithmetic against a restatement
of the reference's eval_wikitext2 loop."""
import ctypes
import math
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import logprob_ref as R  # noqa: E402

F16, BF16, F32 = 1, 2, 0
CODE = {torch.float16: F16, torch.bfloat16: BF16}
E_INVALID, E_UNSUPPORTED = -1, -2
VP, I, I64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_lm_logprob_workspace_bytes.restype = ctypes.c_size_t
    lib.hqq_b200_lm_logprob_workspace_bytes.argtypes = [I64, I64]
    lib.hqq_b200_lm_logprob.argtypes = [VP] * 6 + [I64] * 4 + [I, VP]
    yield lib
    os.environ.pop("HQQ_B200_GEMM_CTAS", None)
    lib.hqq_b200_reload_env()


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def cap(lib, n):
    os.environ["HQQ_B200_GEMM_CTAS"] = str(n)
    lib.hqq_b200_reload_env()


def run(lib, x, W, targets, index_offset=0):
    M, N, K = x.shape[0], W.shape[0], x.shape[1]
    nb = int(lib.hqq_b200_lm_logprob_workspace_bytes(M, N))
    assert nb == -(-N // 128) * M * 8
    ws = torch.full((nb // 4,), float("nan"), dtype=torch.float32)  # scratch arrives dirty
    lse = torch.full((M,), float("nan"), dtype=torch.float32)
    tgt = torch.full((M,), float("nan"), dtype=torch.float32)
    rc = lib.hqq_b200_lm_logprob(P(x), P(W), P(targets), P(lse), P(tgt), P(ws), M, N, K, index_offset, CODE[x.dtype], None)
    assert rc == 0, lib.hqq_b200_last_error()
    return lse, tgt


def make(dtype, M, N, K, seed, index_offset=0):
    """x ~ N(0, 1), W ~ N(0, 4 / K): logits of standard deviation about 2; targets mix -1, 0, N - 1, the shard's inside and outside."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dtype)
    W = (torch.randn(N, K, generator=g) * (2.0 / math.sqrt(K))).to(dtype)
    lo, hi = index_offset, index_offset + N
    pool = torch.tensor([-1, lo, hi - 1, lo - 1, hi, lo + N // 2])
    t = torch.randint(lo, hi, (M,), generator=g)
    pick = torch.randint(0, 2 * len(pool), (M,), generator=g)
    t = torch.where(pick < len(pool), pool[pick.clamp_max(len(pool) - 1)], t)
    return x, W, t.to(torch.int64)


def check(lse, tgt, x, W, targets, index_offset):
    ref_lse, ref_tgt, L, absdot = R.reference(x, W, targets, index_offset)
    b_lse, b_tgt = R.bounds(x, W, targets, index_offset, L, absdot, ref_lse)
    e_lse = (lse.double() - ref_lse).abs()
    assert bool((e_lse <= b_lse).all()), f"lse off by {float((e_lse - b_lse).max()):.3g} past the bound"
    out = ref_tgt.isinf()
    assert bool((tgt[out] == -math.inf).all())
    e_tgt = (tgt.double()[~out] - ref_tgt[~out]).abs()
    assert bool((e_tgt <= b_tgt[~out]).all())


CASES = [(N, M) for N in (128, 1000, 16032) for M in (1, 17, 64, 130)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("ctas", [1, 3])
@pytest.mark.parametrize("N,M", CASES)
def test_lse_head_within_the_float64_bound(emu, dtype, ctas, N, M):
    cap(emu, ctas)
    K = 128 if N < 16032 else 64
    off = 0 if N != 1000 else 5000  # a shard that does not start at row 0
    x, W, t = make(dtype, M, N, K, seed=N * 7 + M, index_offset=off)
    lse, tgt = run(emu, x, W, t, off)
    check(lse, tgt, x, W, t, off)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_a_position_is_the_same_whatever_surrounds_it(emu, dtype):
    """Rows 0..4 of one x, run alone, inside M = 17 and M = 130 blocks at other offsets, under grid caps 1 and 3: identical bits."""
    N, K = 1000, 128
    x, W, t = make(dtype, 130, N, K, seed=11)
    cap(emu, 3)
    base_lse, base_tgt = run(emu, x[:5].contiguous(), W, t[:5].contiguous())
    for ctas in (1, 3):
        cap(emu, ctas)
        for M, at in ((17, 9), (130, 100), (130, 0)):
            g = torch.Generator().manual_seed(M + at)
            xx = torch.randn(M, K, generator=g).to(dtype)
            tt = torch.randint(0, N, (M,), generator=g)
            xx[at:at + 5], tt[at:at + 5] = x[:5], t[:5]
            lse, tgt = run(emu, xx, W, tt)
            assert torch.equal(lse[at:at + 5], base_lse) and torch.equal(tgt[at:at + 5], base_tgt), (ctas, M, at)


@pytest.mark.parametrize("defect", ["target_off_by_one", "drop_tile", "no_mask", "no_rescale"])
def test_planted_defects_leave_the_bound(emu, defect):
    """The kernel's reduction restated in float32 stays inside the bound; each defect leaves it (so the bound is tight enough to see
    it) on the fp16 cases with a ragged vocabulary tile."""
    left = False
    for N, M in ((1000, 130), (130, 64)):
        x, W, t = make(torch.float16, M, N, 128, seed=N + M)
        t = torch.where(t == -1, torch.zeros_like(t), t).clamp(0, N - 1)  # every target inside the shard
        ref_lse, ref_tgt, L, absdot = R.reference(x, W, t, 0)
        b_lse, b_tgt = R.bounds(x, W, t, 0, L, absdot, ref_lse)
        ok_lse, ok_tgt = R.model(L, t, 0)
        assert bool(((ok_lse - ref_lse).abs() <= b_lse).all()) and bool(((ok_tgt - ref_tgt).abs() <= b_tgt).all())
        d_lse, d_tgt = R.model(L, t, 0, defect)
        e_tgt = (d_tgt - ref_tgt).abs().nan_to_num(math.inf)
        left |= bool(((d_lse - ref_lse).abs() > b_lse).any()) or bool((e_tgt > b_tgt).any())
    assert left, defect


def test_bad_arguments(emu):
    x, W, t = make(torch.float16, 4, 128, 64, seed=1)
    lse, tgt = torch.empty(4), torch.empty(4)
    ws = torch.empty(1024)
    call = lambda *a: emu.hqq_b200_lm_logprob(*a)
    ok = (P(x), P(W), P(t), P(lse), P(tgt), P(ws), 4, 128, 64, 0, F16, None)
    assert call(*ok) == 0
    for i in range(6):  # each pointer null
        a = list(ok)
        a[i] = None
        assert call(*a) == E_INVALID
    xb = torch.empty(4 * 64 + 1, dtype=torch.float16)
    a = list(ok)
    a[0] = ctypes.c_void_p(xb.data_ptr() + 2)  # x not 16-byte aligned
    assert call(*a) == E_INVALID
    a = list(ok)
    a[5] = ctypes.c_void_p(ws.data_ptr() + 4)  # workspace not 8-byte aligned
    assert call(*a) == E_INVALID
    a = list(ok)
    a[8] = 60  # K % 8
    assert call(*a) == E_INVALID
    a = list(ok)
    a[6] = 0  # M
    assert call(*a) == E_INVALID
    a = list(ok)
    a[10] = F32
    assert call(*a) == E_UNSUPPORTED


def eval_wikitext2_windows(seq_len, max_length, stride):
    """The window loop of the reference's examples/llama2_benchmark/eval_model.py::eval_wikitext2, restated: per window (begin,
    end, trg_len, the indices of the shifted labels its loss averages over), and the end_loc its perplexity divides by."""
    out = []
    for i in range(0, seq_len, stride):
        begin_loc = max(i + stride - max_length, 0)
        end_loc = min(i + stride, seq_len)
        trg_len = end_loc - i
        target_ids = torch.arange(begin_loc, end_loc)
        target_ids[:-trg_len] = -100
        shifted = target_ids[1:]  # the causal LM loss: logits[j] predicts labels[j + 1]
        kept = torch.nonzero(shifted != -100).flatten().tolist()
        out.append((begin_loc, end_loc, trg_len, kept))
    return out, end_loc


@pytest.mark.parametrize("seq_len,max_length,stride", [(5000, 1024, 512), (1024, 1024, 512), (1025, 1024, 512), (100, 1024, 512),
                                                       (3000, 256, 100), (2048, 1024, 1024), (7, 4, 3), (9, 2, 5)])
def test_perplexity_windows_follow_the_reference_loop(seq_len, max_length, stride):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    import perplexity
    want, end = eval_wikitext2_windows(seq_len, max_length, stride)
    got = perplexity.windows(seq_len, max_length, stride)
    assert [(w.begin, w.end, w.trg_len, list(range(*w.scored()))) for w in got] == want
    assert got[-1].end == end


def test_perplexity_of_window_logprobs_restates_the_reference():
    """eval_wikitext2: ll_w = trg_len * mean(-log p over the window's kept labels); ppl = exp(sum ll / end_loc)."""
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    import perplexity
    g = torch.Generator().manual_seed(3)
    want_w, end_loc = eval_wikitext2_windows(3000, 1024, 512)
    wins = perplexity.windows(3000, 1024, 512)
    lps = [-torch.rand(w.end - w.begin - 1, generator=g, dtype=torch.float64) * 5 for w in wins]
    lls = [-lp[kept].mean() * trg_len for (_, _, trg_len, kept), lp in zip(want_w, lps)]
    want = math.exp(float(torch.stack(lls).sum()) / end_loc)
    assert perplexity.perplexity(wins, lps) == pytest.approx(want, rel=1e-12)
