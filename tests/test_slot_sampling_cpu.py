"""Per-slot sampling on the CPU kernel emulator: hqq_b200_glue_penalize against the fp32 restatement of tests/penalty_ref.py (bit
for bit, counts included), hqq_b200_glue_sample_slots against hqq_b200_glue_sample / _pos, the framework-op restatements the
fused=False model uses, argument checks and the rejected model options."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import penalty_ref  # noqa: E402
from hqq_b200 import harness  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
E_INVALID = -1
VP, I, F, U64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_uint64
SEED = 0x0BAD_5EED_1234_5678


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_glue_sample.argtypes = [VP, I, I, I, F, I, F, U64, VP, VP, I, VP]
    lib.hqq_b200_glue_sample_pos.argtypes = [VP, I, I, I, F, I, F, U64, I, VP, VP, VP, I, VP]
    lib.hqq_b200_glue_sample_slots.argtypes = [VP, I, I, I, I, VP, VP, VP, U64, VP, VP, VP, VP, I, VP]
    lib.hqq_b200_glue_penalize.argtypes = [VP, I, I, I, I] + [VP] * 7 + [I, I, VP]
    return lib


def p(t):
    return VP(t.data_ptr()) if t is not None else None


def penalize(emu, x, n, T, rep, freq, pres, counts, prompt, tok, dtype):
    """The kernel on x[:, :n] (x [rows, ld]); returns (out [rows, n], counts after)."""
    rows, ld = x.shape
    ld_out = -(-n // 8) * 8
    out = torch.full((rows, ld_out), float("nan"), dtype=dtype)
    counts = counts.clone()
    rc = emu.hqq_b200_glue_penalize(p(x), n, ld, rows, T, p(rep), p(freq), p(pres), p(counts), p(prompt), p(tok), p(out), ld_out, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out[:, :n], counts


def bits(t):
    return t.view(torch.int16)


def special_rows(gen, rows, ld, dtype):
    """Normal logits with negatives, exact zeros, -0, +-inf, large magnitudes and values at the dtype's edges."""
    x = torch.randn(rows, ld, generator=gen, dtype=torch.float64) * 4
    x = x.to(dtype)
    flat = x.view(-1)
    m = flat.numel()
    idx = torch.randperm(m, generator=gen)
    specials = [0.0, -0.0, float("inf"), float("-inf"), 1e-7, -1e-7, 60000.0 if dtype == torch.float16 else 3e38, -1.0, 1.0]
    for j, v in enumerate(specials * 4):
        flat[idx[j]] = v
    return x


def tables(gen, slots, n):
    """counts with 0 / 1 / many entries and prompt flags, some only in the prompt."""
    u = torch.rand(slots, n, generator=gen)
    counts = torch.where(u < 0.6, 0, torch.where(u < 0.8, 1, torch.randint(2, 40, (slots, n), generator=gen))).to(torch.int32)
    prompt = (torch.rand(slots, n, generator=gen) < 0.3).to(torch.uint8)
    return counts, prompt


def params(slots, neutral_slot=None):
    rep = torch.tensor([1.3, 0.7, 1.0, 2.5, 1.1, 1.05, 0.9, 1.7][:slots], dtype=torch.float32)
    freq = torch.tensor([0.5, -0.25, 0.0, 1.0, 0.1, 0.0, 0.3, 2.0][:slots], dtype=torch.float32)
    pres = torch.tensor([0.25, 0.0, 0.0, -0.5, 0.6, 1.5, 0.0, 0.2][:slots], dtype=torch.float32)
    if neutral_slot is not None:
        rep[neutral_slot], freq[neutral_slot], pres[neutral_slot] = 1.0, 0.0, 0.0
    return rep, freq, pres


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_penalize_is_bit_exact(emu, dtype):
    gen = torch.Generator().manual_seed(100 + CODE[dtype])
    for n, T, slots in ((7, 1, 3), (1000, 2, 4), (2049, 4, 2), (1031, 1, 8), (3000, 8, 1)):
        rows = slots * T
        x = special_rows(gen, rows, n + 5, dtype)  # ld not a multiple of 8: the input rows need no alignment
        counts, prompt = tables(gen, slots, n)
        rep, freq, pres = params(slots, neutral_slot=slots - 1 if slots > 1 else None)
        tok = torch.randint(0, n, (slots,), generator=gen)
        if slots > 2:
            tok[1] = -1   # nothing to count
            tok[2] = n    # outside the vocabulary: nothing to count
        for t in (tok, None):
            got, gc = penalize(emu, x, n, T, rep, freq, pres, counts, prompt, t, dtype)
            ref, rc = penalty_ref.penalize(x[:, :n], T, rep, freq, pres, counts, prompt, t)
            assert torch.equal(bits(got), bits(ref)), (n, T, slots, (bits(got) != bits(ref)).nonzero()[:5])
            assert torch.equal(gc, rc), (n, T, slots)
            # the model's own restatement (fused=False) agrees on one row per slot
            if T == 1:
                h = harness.apply_penalties(x[:, :n], rc, prompt, rep, freq, pres)
                assert torch.equal(bits(h), bits(ref))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_penalize_neutral_keeps_every_bit(emu, dtype):
    """r = 1, f = p = 0 on rows where every element is seen and counted: the output bits are the input bits (-0, +-inf included)."""
    gen = torch.Generator().manual_seed(200 + CODE[dtype])
    n, slots, T = 1500, 3, 2
    x = special_rows(gen, slots * T, n, dtype)
    counts = torch.randint(1, 9, (slots, n), generator=gen).to(torch.int32)
    prompt = torch.ones(slots, n, dtype=torch.uint8)
    one, zero = torch.ones(slots), torch.zeros(slots)
    got, gc = penalize(emu, x, n, T, one, zero, zero, counts, prompt, torch.tensor([0, 5, n - 1]), dtype)
    assert torch.equal(bits(got), bits(x))
    assert int((gc - counts).sum()) == 3


def test_emulated_penalize_counts_the_token_before_its_own_row(emu):
    """tok[b] is counted once per slot (all rows_per_slot rows see the incremented count), before the penalty: a token never seen
    before takes the presence and frequency penalties of count 1 in the step that consumes it."""
    n, T, slots = 2100, 4, 2
    x = torch.full((slots * T, n), 2.0, dtype=torch.float16)
    counts = torch.zeros(slots, n, dtype=torch.int32)
    counts[1, 7] = 3
    prompt = torch.zeros(slots, n, dtype=torch.uint8)
    rep, freq, pres = torch.tensor([2.0, 1.0]), torch.tensor([0.5, 0.5]), torch.tensor([0.25, 0.0])
    tok = torch.tensor([2050, 7])  # slot 0's token in the third column chunk
    got, gc = penalize(emu, x, n, T, rep, freq, pres, counts, prompt, tok, torch.float16)
    assert int(gc[0, 2050]) == 1 and int(gc[1, 7]) == 4 and int(gc.sum()) == 5
    assert torch.all(got[:T, 2050] == (2.0 / 2.0 - 0.5) - 0.25)   # count 1: this step's token
    assert torch.all(got[T:, 7] == 2.0 - 0.5 * 4)
    assert torch.equal(got[:T, :2050], x[:T, :2050]) and torch.equal(got[T:, 8:], x[T:, 8:])
    # without tok (a prefill head) nothing is counted and the penalties use the counts as they are
    got, gc = penalize(emu, x, n, T, rep, freq, pres, counts, prompt, None, torch.float16)
    assert torch.equal(gc, counts) and torch.all(got[:T, 2050] == 2.0) and torch.all(got[T:, 7] == 2.0 - 0.5 * 3)


def sample(emu, x, n, Tm, k, pp, ctr=None, pos=None, seq=None, T=1, dtype=torch.float16):
    rows, ld = x.shape
    out = torch.full((rows,), -1, dtype=torch.int64)
    if pos is None:
        rc = emu.hqq_b200_glue_sample(p(x), n, ld, rows, Tm, k, pp, SEED, p(ctr), p(out), CODE[dtype], None)
    else:
        rc = emu.hqq_b200_glue_sample_pos(p(x), n, ld, rows, Tm, k, pp, SEED, T, p(pos), p(seq), p(out), CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out


def sample_slots(emu, x, n, temp, topk, topp, ctr=None, pos=None, seq=None, T=1, dtype=torch.float16):
    rows, ld = x.shape
    out = torch.full((rows,), -1, dtype=torch.int64)
    rc = emu.hqq_b200_glue_sample_slots(p(x), n, ld, rows, T, p(temp), p(topk), p(topp), SEED, p(ctr), p(pos), p(seq), p(out), CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out


def slot_params(slots, Tm, k, pp):
    return (torch.full((slots,), Tm, dtype=torch.float32), torch.full((slots,), k, dtype=torch.int32), torch.full((slots,), pp, dtype=torch.float32))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_sample_slots_is_the_shared_sampler(emu, dtype):
    """Every slot on the same parameters: the tokens of hqq_b200_glue_sample (step keys) and hqq_b200_glue_sample_pos (position keys)."""
    gen = torch.Generator().manual_seed(300 + CODE[dtype])
    for n, (Tm, k, pp) in ((1000, (0.6, 5, 1.0)), (4097, (1.0, 0, 0.9)), (64, (0.7, 50, 0.95)), (2048, (2.0, 0, 1.0))):
        rows = 4
        x = (torch.randn(rows, -(-n // 8) * 8, generator=gen, dtype=torch.float64) * 2.5).to(dtype)
        ctr = torch.tensor([2 ** 32 + 5], dtype=torch.int64)
        ref = sample(emu, x, n, Tm, k, pp, ctr=ctr, dtype=dtype)
        assert torch.equal(sample_slots(emu, x, n, *slot_params(rows, Tm, k, pp), ctr=ctr, dtype=dtype), ref)
        for T in (1, 2):
            pos, seq = torch.tensor([3, 900][: rows // T] + [17] * 4)[: rows // T], torch.tensor([1, 2 ** 31 - 1, 5, 6])[: rows // T]
            ref = sample(emu, x, n, Tm, k, pp, pos=pos, seq=seq, T=T, dtype=dtype)
            got = sample_slots(emu, x, n, *slot_params(rows // T, Tm, k, pp), pos=pos, seq=seq, T=T, dtype=dtype)
            assert torch.equal(got, ref), (n, T)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_sample_slots_mixed_rows(emu, dtype):
    """Rows at temperature 0 give torch.argmax (first index on ties, -0 equal to +0); the other rows are the rows the scalar
    sampler draws with their own parameters, at their own row index."""
    gen = torch.Generator().manual_seed(400 + CODE[dtype])
    n, rows = 1500, 5
    x = (torch.randn(rows, 1504, generator=gen, dtype=torch.float64) * 2).to(dtype)
    x[0, [10, 700, 1400]] = 9.0          # ties at the maximum: the first index wins
    x[2, :n] = 0.0
    x[2, 3] = -0.0                       # all zero: index 0
    x[4, 5] = float("inf")
    temp = torch.tensor([0.0, 0.8, 0.0, 1.3, 0.0])
    topk = torch.tensor([0, 5, 3, 0, 7], dtype=torch.int32)
    topp = torch.tensor([1.0, 0.9, 0.5, 1.0, 1.0])
    ctr = torch.tensor([9], dtype=torch.int64)
    got = sample_slots(emu, x, n, temp, topk, topp, ctr=ctr, dtype=dtype)
    arg = torch.argmax(x[:, :n], dim=-1)
    assert [int(got[b]) for b in (0, 2, 4)] == [int(arg[b]) for b in (0, 2, 4)] == [10, 0, 5]
    for b in (1, 3):
        ref = sample(emu, x, n, float(temp[b]), int(topk[b]), float(topp[b]), ctr=ctr, dtype=dtype)
        assert int(got[b]) == int(ref[b])
    # the framework-op restatement with per-row tensors: the same argmax rows, and sample_tokens' scalar tokens row by row
    ref_rows = harness.sample_tokens(x[:, :n], temp, topk, topp, SEED, ctr)
    assert [int(ref_rows[b]) for b in (0, 2, 4)] == [10, 0, 5]
    for b in (1, 3):
        assert int(ref_rows[b]) == int(harness.sample_tokens(x[:, :n], float(temp[b]), int(topk[b]), float(topp[b]), SEED, ctr)[b])


def test_sample_tokens_with_per_row_tensors_matches_the_scalar_form():
    """sample_tokens with every row on the same tensor parameters draws the scalar form's tokens (step and position counters)."""
    gen = torch.Generator().manual_seed(17)
    x = (torch.randn(6, 3000, generator=gen, dtype=torch.float64) * 3).to(torch.float16)
    x[:, 100:140] = x[:, 100:101]  # ties at a pivot
    ctr = torch.tensor([12], dtype=torch.int64)
    pc = harness.position_counter(torch.arange(6) * 7, torch.tensor([1, 1, 2, 3, 5, 8]))
    for Tm, k, pp in ((0.6, 5, 1.0), (1.0, 0, 0.9), (0.7, 50, 0.95), (2.0, 0, 1e-3), (1.0, 3000, 0.5), (0.25, 1, 1.0)):
        t = slot_params(6, Tm, k, pp)
        for c in (ctr, pc):
            assert torch.equal(harness.sample_tokens(x, *t, SEED, c), harness.sample_tokens(x, Tm, k, pp, SEED, c)), (Tm, k, pp)


def test_emulated_penalize_and_sample_slots_argument_checks(emu):
    x = torch.zeros(4, 64, dtype=torch.float16)
    out = torch.zeros(4, 64, dtype=torch.float16)
    f = torch.ones(4)
    counts, prompt = torch.zeros(4, 64, dtype=torch.int32), torch.zeros(4, 64, dtype=torch.uint8)
    tok = torch.zeros(4, dtype=torch.int64)

    def pen(n=64, ld=64, rows=4, T=1, rep=f, counts=counts, prompt=prompt, out_ptr=None, ld_out=64, dtype=F16):
        o = out_ptr if out_ptr is not None else out.data_ptr()
        return emu.hqq_b200_glue_penalize(p(x), n, ld, rows, T, p(rep), p(f), p(f), p(counts), p(prompt), p(tok), VP(o), ld_out, dtype, None)

    assert pen() == 0 and pen(T=2) == 0 and pen(T=4) == 0
    for kw in (dict(n=0), dict(ld=63), dict(ld_out=60, n=60), dict(ld_out=56), dict(rows=0), dict(T=0), dict(T=3), dict(T=16, rows=16), dict(rep=None),
               dict(counts=None), dict(prompt=None), dict(out_ptr=out.data_ptr() + 2), dict(out_ptr=x.data_ptr()), dict(out_ptr=x.data_ptr() + 64),
               dict(dtype=0)):
        assert pen(**kw) == E_INVALID, kw
        assert b"hqq_b200_glue_penalize" in emu.hqq_b200_last_error(), kw

    temp, topk, topp = slot_params(4, 1.0, 0, 1.0)
    ctr, pos, seq = torch.zeros(1, dtype=torch.int64), torch.zeros(4, dtype=torch.int64), torch.zeros(4, dtype=torch.int64)
    res = torch.zeros(4, dtype=torch.int64)

    def smp(n=64, ld=64, rows=4, T=1, temp=temp, ctr=ctr, pos=None, seq=None, xp=None, dtype=F16):
        return emu.hqq_b200_glue_sample_slots(VP(xp or x.data_ptr()), n, ld, rows, T, p(temp), p(topk), p(topp), SEED, p(ctr), p(pos), p(seq), p(res),
                                              dtype, None)

    assert smp() == 0 and smp(ctr=None, pos=pos, seq=seq) == 0 and smp(T=2) == 0
    for kw in (dict(ctr=None), dict(ctr=None, pos=pos), dict(temp=None), dict(n=0), dict(ld=60, n=60), dict(ld=63), dict(rows=0), dict(T=3),
               dict(T=0), dict(xp=x.data_ptr() + 2), dict(dtype=0)):
        assert smp(**kw) == E_INVALID, kw
        assert b"hqq_b200_glue_sample_slots" in emu.hqq_b200_last_error(), kw


def test_slot_sampling_with_spec_k_is_rejected_before_any_weight():
    with pytest.raises(ValueError, match="slot_sampling cannot be combined with spec_k"):
        harness.DecodeModel(harness.LLAMA3_8B, n_layers=1, device="cpu", ragged=True, spec_k=2, slot_sampling=True)
    with pytest.raises(ValueError, match="slot_sampling cannot be combined with spec_k"):
        harness.DecodeModel(harness.LLAMA3_8B, n_layers=1, device="cpu", ragged=True, spec_k=2, slot_sampling=True, do_sample=True,
                            sample_keys="position")
