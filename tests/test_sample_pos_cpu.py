"""hqq_b200_glue_sample_pos (csrc/decode_glue.cu) on the CPU kernel emulator against sample_tokens with per-row counters.

Row r of a launch is slot b = r / T at position pos[b] + r % T.  The float64 restatement of row r is sample_tokens on the rows of
window offset t = r % T, one per slot (row index b), with position_counter(pos + t, seq).  Every token must be the float64 token or
lie in the set tests/sample_ref.py accepts; planted defects in the counter words must each change a token of the grid.  A
chi-square test checks, on the restatement, that accepting drafts while they equal the sampled targets and emitting the first
target that differs gives every emitted position the kept softmax of its row."""
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
import sample_ref as S  # noqa: E402
import spec_ref  # noqa: E402
from hqq_b200 import harness  # noqa: E402
from hqq_b200.harness import philox_uniforms, position_counter, sample_tokens  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
E_INVALID = -1
VP, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
SEED = 0x0F1E_2D3C_4B5A_6978


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_glue_sample_pos.argtypes = [VP, I, I, I, F, I, F, ctypes.c_uint64, I, VP, VP, VP, I, VP]
    return lib


def run(emu, x, n, T, temp, k, p, pos, seq, dtype):
    """x [B T, ld] in dtype; the kernel's tokens for x[:, :n], rows_per_slot T."""
    rows, ld = x.shape
    pt, st = torch.tensor(pos, dtype=torch.int64), torch.tensor(seq, dtype=torch.int64)
    out = torch.full((rows,), -1, dtype=torch.int64)
    rc = emu.hqq_b200_glue_sample_pos(VP(x.data_ptr()), n, ld, rows, temp, k, p, SEED, T, VP(pt.data_ptr()), VP(st.data_ptr()), VP(out.data_ptr()),
                                      CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out


def window_rows(x, n, T, t):
    """The rows of window offset t, one per slot: [B, n]."""
    return x.view(-1, T, x.shape[1])[:, t, :n]


# (n, T, temperature, top_k, top_p, pos, seq): one pos / seq entry per slot.  Positions 0, 63, 64 and 131071 with the window
# offsets crossing 64 and passing 131071; full-vocabulary rows, the costly ones to emulate, in one case (the GPU test runs more)
P0, P63, P64, PMAX = 0, 63, 64, 131071
S_MAX = 2 ** 31 - 1
CASES = [(1, 1, 0.6, 5, 1.0, [P0, P63], [0, 1]), (1, 8, 1.0, 0, 0.9, [P64, PMAX], [S_MAX, 0]), (7, 4, 0.6, 5, 1.0, [P63, P0], [1, S_MAX]),
         (7, 8, 2.0, 0, 0.5, [PMAX, P64], [0, 1]), (7, 1, 0.25, 50, 0.95, [P0, P63], [S_MAX, 0]), (1000, 1, 0.6, 5, 1.0, [P64, PMAX], [1, S_MAX]),
         (1000, 4, 1.0, 0, 0.9, [P63, P0], [0, 1]), (1000, 8, 0.7, 50, 0.95, [PMAX, P64], [S_MAX, 0]),
         (128256, 1, 0.6, 5, 1.0, [PMAX, P64], [1, S_MAX])]
DEFECTS = ["slot and row swapped", "t dropped from the position", "seq word dropped", "high bit missing"]


def defect_uniforms(name, n, B, T, t, pos, seq):
    """Uniforms [B, n] of window offset t under a planted defect of the counter words."""
    p, s = torch.tensor(pos) + (0 if name == "t dropped from the position" else t), torch.tensor(seq)
    ctr = position_counter(p, s)
    if name == "seq word dropped":
        ctr[:, 1] = 0x80000000
    elif name == "high bit missing":
        ctr[:, 1] &= 0x7FFFFFFF
    if name == "slot and row swapped":  # word 1 = the row's index in the launch, b T + t
        return philox_uniforms(n, B * T, SEED, ctr.repeat_interleave(T, dim=0)).view(B, T, n)[:, t]
    return philox_uniforms(n, B, SEED, ctr)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_sample_pos_matches_float64_and_defects_change_tokens(emu, dtype):
    gen = torch.Generator().manual_seed(40 + CODE[dtype])
    stats = {"rows": 0, "differ": 0}
    caught = {d: False for d in DEFECTS}
    for n, T, temp, k, p, pos, seq in CASES:
        B = len(pos)
        ld = -(-n // 8) * 8 + 8
        x = (torch.randn(B * T, ld, generator=gen, dtype=torch.float64) * 2.5).to(dtype)
        got = run(emu, x, n, T, temp, k, p, pos, seq, dtype).view(B, T)
        for t in range(T):
            lg = window_rows(x, n, T, t)
            ctr = position_counter(torch.tensor(pos) + t, torch.tensor(seq))
            ref = sample_tokens(lg, temp, k, p, SEED, ctr)
            u = philox_uniforms(n, B, SEED, ctr)
            assert torch.equal(ref, S.restate(lg, temp, k, p, u)), "the two float64 restatements disagree"
            for b, (t0, ok, why) in enumerate(S.accepted(lg, temp, k, p, u)):
                assert t0 == int(ref[b])
                assert int(got[b, t]) in ok, (n, T, t, b, pos[b], seq[b], int(got[b, t]), t0)
                stats["rows"] += 1
                stats["differ"] += int(got[b, t]) != t0
                if len(ok) > 1:
                    stats[why] = stats.get(why, 0) + 1
            for d in DEFECTS:
                if not caught[d] and not torch.equal(S.restate(lg, temp, k, p, defect_uniforms(d, n, B, T, t, pos, seq)), got[:, t]):
                    caught[d] = True
    print(f"{dtype}: {stats}")
    assert stats["differ"] <= stats["rows"] // 50, stats
    assert all(caught.values()), caught


def test_emulated_sample_pos_row_invariance(emu):
    """A row's token depends on its bits, the parameters, seed, slot, position and seq alone: slot 0 launched without slot 1, or
    next to a slot 1 with other rows, position and seq, and a launch with T = 1 whose pos lists each row's position, give the same
    tokens."""
    gen = torch.Generator().manual_seed(3)
    n, T = 1000, 4
    x = (torch.randn(2 * T, 1024, generator=gen, dtype=torch.float64) * 2.5).to(torch.float16)
    a = run(emu, x, n, T, 0.8, 0, 0.9, [10, 500], [3, 4], torch.float16)
    assert torch.equal(run(emu, x[:T].clone(), n, T, 0.8, 0, 0.9, [10], [3], torch.float16), a[:T])
    y = x.clone()
    y[T:] = torch.flip(x[T:], dims=[1])
    assert torch.equal(run(emu, y, n, T, 0.8, 0, 0.9, [10, 7], [3, 9], torch.float16)[:T], a[:T])
    for t in range(T):  # window offset t as a T = 1 launch: rows at positions pos + t, one per slot
        rows = window_rows(x, 1024, T, t).contiguous()
        assert torch.equal(run(emu, rows, n, 1, 0.8, 0, 0.9, [10 + t, 500 + t], [3, 4], torch.float16), a.view(2, T)[:, t])


def test_emulated_sample_pos_argument_checks(emu):
    x = torch.zeros(4, 64, dtype=torch.float16)
    pos, seq = torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int64)
    out = torch.zeros(4, dtype=torch.int64)

    def call(n=64, ld=64, rows=4, temp=1.0, k=0, p=1.0, T=2, ptr=None, dtype=F16, nulls=()):
        a = {"pos": pos.data_ptr(), "seq": seq.data_ptr(), "out": out.data_ptr()}
        for z in nulls:
            a[z] = None
        return emu.hqq_b200_glue_sample_pos(VP(ptr if ptr is not None else x.data_ptr()), n, ld, rows, temp, k, p, 0, T, VP(a["pos"]), VP(a["seq"]),
                                            VP(a["out"]), dtype, None)

    assert call() == 0
    bad = [dict(temp=0.0), dict(temp=float("nan")), dict(k=-1), dict(p=0.0), dict(p=1.5), dict(n=0), dict(ld=63, n=64), dict(rows=0), dict(rows=3),
           dict(T=0), dict(T=9, rows=9), dict(T=-1), dict(ld=60, n=60), dict(ptr=x.data_ptr() + 2), dict(dtype=0), dict(ptr=0),
           dict(nulls=("pos",)), dict(nulls=("seq",)), dict(nulls=("out",))]
    for kw in bad:
        assert call(**kw) == E_INVALID, kw
        assert b"hqq_b200_glue_sample_pos" in emu.hqq_b200_last_error(), kw


def test_equality_accept_gives_the_marginal_chi_square():
    """Targets drawn by sample_tokens at each window row's position keys, drafts fixed: with spec_ref.accept, the token emitted at
    window offset j (when the stream reaches it) follows row j's kept softmax, for every j -- single-token drafts make
    equality-accept exact speculative sampling.  The draws differ by slot (Philox word 1) and sequence number."""
    from scipy.stats import chisquare
    n, K, R = 8, 3, 20000
    temp, top_k, top_p = 0.6, 5, 1.0
    gen = torch.Generator().manual_seed(5)
    rows = (torch.randn(K + 1, n, generator=gen, dtype=torch.float64) * 1.2).to(torch.float16)
    drafts = [int(rows[j].double().argmax()) for j in range(K)]  # the likeliest tokens: many streams reach every offset
    pos0, seq = 1000, torch.arange(R) % 7
    targets = torch.stack([sample_tokens(rows[t].view(1, n).expand(R, n), temp, top_k, top_p, SEED,
                                         position_counter(torch.full((R,), pos0 + t), seq)) for t in range(K + 1)], dim=1).tolist()
    emitted = [spec_ref.accept(0, drafts, targets[r], pos0, 1 << 17)[0] for r in range(R)]
    for j in range(K + 1):
        lv = rows[j].double().view(1, n)
        keep = S.keep_topp(lv, S.keep_topk(lv, top_k), S.fp32(temp), S.fp32(top_p))[0]
        w = torch.where(keep, torch.exp((lv[0] - lv[0].max()) / S.fp32(temp)), torch.zeros(n, dtype=torch.float64))
        prob = w / w.sum()
        got = [e[j] for e in emitted if len(e) > j]
        counts = torch.bincount(torch.tensor(got), minlength=n).double()
        assert counts[~keep].sum() == 0
        assert len(got) >= 1000, (j, len(got))
        stat, pval = chisquare(counts[keep].numpy(), (prob[keep] * len(got)).numpy())
        print(f"offset {j}: {len(got)} streams, chi2 {stat:.1f}, p {pval:.3g}")
        assert pval >= 1e-4, (j, pval)


def test_position_keys_options_rejected():
    """sample_keys other than "step" / "position", position keys without do_sample, and spec_k with do_sample under step keys raise
    ValueError (before any device work)."""
    for kw in (dict(sample_keys="row"), dict(sample_keys="position"), dict(sample_keys="position", do_sample=False),
               dict(do_sample=True, spec_k=2, ragged=True), dict(do_sample=True, sample_keys="step", spec_k=2, ragged=True)):
        with pytest.raises(ValueError):
            harness.DecodeModel(harness.LLAMA3_8B, n_layers=1, device="cpu", **kw)
