"""hqq_b200_glue_sample (csrc/decode_glue.cu) on the CPU kernel emulator against the float64 restatement.

Every token must be the float64 token of sample_tokens, or lie in the set tests/sample_ref.py accepts where the kernel's fp32
arithmetic may order two candidates the other way (race keys within their error bound, a top-p boundary within the fixed-point
mass error); how often that set is needed is counted and printed.  Planted defects, made on the same uniforms, must each change a
token of the grid."""
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
from hqq_b200.harness import philox_uniforms, sample_tokens  # noqa: E402

F16, BF16 = 1, 2
CODE = {torch.float16: F16, torch.bfloat16: BF16}
E_INVALID = -1
VP, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
SEED = 0x1234_5678_9ABC_DEF0


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_glue_sample.argtypes = [VP, I, I, I, F, I, F, ctypes.c_uint64, VP, VP, I, VP]
    return lib


def run(emu, x, n, T, k, p, seed, ctr, dtype):
    """x [rows, ld] in dtype; the kernel's tokens for x[:, :n]."""
    rows, ld = x.shape
    c = torch.tensor([ctr], dtype=torch.int64)
    out = torch.full((rows,), -1, dtype=torch.int64)
    rc = emu.hqq_b200_glue_sample(VP(x.data_ptr()), n, ld, rows, T, k, p, seed, VP(c.data_ptr()), VP(out.data_ptr()), CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return out


def row_block(gen, rows, n, dtype, ties=False):
    ld = -(-n // 8) * 8 + 8
    if ties:  # few distinct values: many elements share the top-k pivot and the top-p threshold
        x = torch.randint(-6, 3, (rows, ld), generator=gen).double() * 0.5
    else:
        x = torch.randn(rows, ld, generator=gen, dtype=torch.float64) * 2.5
    return x.to(dtype)


NS = [1, 7, 8, 1000, 4097, 128256]
COUNTERS = [0, 1, 2 ** 32 + 7, 2 ** 40 + 2 ** 32 - 1]


def combos(n):
    """(T, top_k, top_p) covering T {0.25, 0.6, 1, 2}, top_k {0, 1, 5, 50, n, n + 1}, top_p {1, 0.9, 0.5, 1e-3}."""
    return [(0.25, 0, 1.0), (0.6, 5, 1.0), (1.0, 0, 0.9), (2.0, 50, 0.5), (0.6, 1, 1e-3), (1.0, n, 0.9), (0.25, n + 1, 0.5), (0.7, 50, 0.95),
            (2.0, 0, 1e-3), (0.6, 5, 0.9)]


def check_case(x, n, T, k, p, ctr, got, stats):
    logits = x[:, :n]
    u = philox_uniforms(n, x.shape[0], SEED, ctr)
    ref = sample_tokens(logits, T, k, p, SEED, ctr)
    assert torch.equal(ref, S.restate(logits, T, k, p, u)), "the two float64 restatements disagree"
    for b, (t0, ok, why) in enumerate(S.accepted(logits, T, k, p, u)):
        assert t0 == int(ref[b])
        assert int(got[b]) in ok, (n, T, k, p, ctr, b, int(got[b]), t0, sorted(ok)[:8])
        stats["rows"] += 1
        if len(ok) > 1:
            stats[why] = stats.get(why, 0) + 1
        stats["differ"] += int(got[b]) != t0


DEFECTS = ["temperature ignored", "strict pivot", "philox index + 1", "row dropped from the counter", "top-p before top-k"]


def defect_tokens(name, logits, T, k, p, ctr):
    rows, n = logits.shape
    if name == "philox index + 1":
        u = philox_uniforms(n + 1, rows, SEED, ctr)[:, 1:]
    elif name == "row dropped from the counter":
        u = philox_uniforms(n, 1, SEED, ctr).expand(rows, n)
    else:
        u = philox_uniforms(n, rows, SEED, ctr)
    return S.restate(logits, T, k, p, u, defect=name if name in ("temperature ignored", "strict pivot", "top-p before top-k") else None)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_sample_matches_float64_and_defects_change_tokens(emu, dtype):
    gen = torch.Generator().manual_seed(CODE[dtype])
    stats = {"rows": 0, "differ": 0}
    caught = {d: False for d in DEFECTS}
    i = 0
    for n in NS:
        for T, k, p in combos(n):
            rows = 1 if i % 4 == 3 else 3
            ctr = COUNTERS[i % len(COUNTERS)]
            i += 1
            x = row_block(gen, rows, n, dtype, ties=(i % 5 == 0))
            got = run(emu, x, n, T, k, p, SEED, ctr, dtype)
            check_case(x, n, T, k, p, ctr, got, stats)
            for d in DEFECTS:
                if not caught[d] and not torch.equal(defect_tokens(d, x[:, :n], T, k, p, ctr), got):
                    caught[d] = True
    print(f"{dtype}: {stats}")
    assert stats["differ"] == 0 or stats["differ"] <= stats["rows"] // 50, stats
    assert all(caught.values()), caught


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_emulated_sample_ties_at_the_pivot_and_threshold(emu, dtype):
    """Rows of a few distinct values: every element tied with the top-k pivot stays in the race, and top-p keeps whole tie groups."""
    gen = torch.Generator().manual_seed(7 + CODE[dtype])
    stats = {"rows": 0, "differ": 0}
    n = 4097
    for T, k, p in ((0.6, 5, 1.0), (1.0, 50, 1.0), (1.0, 0, 0.5), (0.7, 50, 0.95), (2.0, 1, 1.0)):
        x = row_block(gen, 3, n, dtype, ties=True)
        for ctr in (3, 2 ** 33):
            got = run(emu, x, n, T, k, p, SEED, ctr, dtype)
            check_case(x, n, T, k, p, ctr, got, stats)
    print(f"{dtype}: {stats}")


def test_emulated_sample_does_not_depend_on_rows_or_stride(emu):
    """Row b's token depends on its bits, n, the parameters, seed, counter and b alone."""
    gen = torch.Generator().manual_seed(11)
    n = 1000
    x = row_block(gen, 3, n, torch.float16)
    a = run(emu, x, n, 0.8, 0, 0.9, SEED, 5, torch.float16)
    wide = torch.zeros(3, 1024 + 64, dtype=torch.float16)
    wide[:, :n] = x[:, :n]
    assert torch.equal(run(emu, wide, n, 0.8, 0, 0.9, SEED, 5, torch.float16), a)
    assert int(run(emu, x[:1].clone(), n, 0.8, 0, 0.9, SEED, 5, torch.float16)[0]) == int(a[0])
    assert torch.equal(run(emu, x, n, 0.8, 0, 0.9, SEED, 5, torch.float16), a)


def test_emulated_top_k_1_is_the_argmax(emu):
    gen = torch.Generator().manual_seed(12)
    for dtype in (torch.float16, torch.bfloat16):
        x = row_block(gen, 3, 4097, dtype)
        got = run(emu, x, 4097, 1.3, 1, 1.0, SEED, 9, dtype)
        assert torch.equal(got, torch.argmax(x[:, :4097].float(), dim=-1))


def test_emulated_sample_argument_checks(emu):
    x = torch.zeros(2, 64, dtype=torch.float16)
    c = torch.zeros(1, dtype=torch.int64)
    out = torch.zeros(2, dtype=torch.int64)

    def call(n=64, ld=64, rows=2, T=1.0, k=0, p=1.0, ptr=None, dtype=F16, counter=True):
        return emu.hqq_b200_glue_sample(VP(ptr if ptr is not None else x.data_ptr()), n, ld, rows, T, k, p, 0, VP(c.data_ptr()) if counter else None,
                                        VP(out.data_ptr()), dtype, None)

    assert call() == 0
    bad = [dict(T=0.0), dict(T=-1.0), dict(T=float("inf")), dict(T=float("nan")), dict(k=-1), dict(p=0.0), dict(p=1.5), dict(p=float("nan")),
           dict(n=0), dict(ld=63, n=64), dict(rows=0), dict(ld=60, n=60), dict(ptr=x.data_ptr() + 2), dict(dtype=0), dict(counter=False)]
    for kw in bad:
        assert call(**kw) == E_INVALID, kw
        assert b"hqq_b200_glue_sample" in emu.hqq_b200_last_error(), kw
