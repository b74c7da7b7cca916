"""The mixture-of-experts kernels on the CPU kernel emulator (tests/emu): the router (hqq_b200_glue_moe_route), the expert-grouped mode
of the small-M kernel (hqq_b200_linear_fwd_grouped) and the combine (hqq_b200_glue_moe_combine), against the restatements of
tests/moe_ref.py and the float64 bound of tests/fused_ref.py; and the argument checks of the decode harness's MoE shapes."""
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
import fused_ref as FR  # noqa: E402
import moe_ref as MR  # noqa: E402

F16, BF16 = 1, 2
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
    lib.hqq_b200_glue_moe_route.argtypes = [VP, VP, I, I, I, I] + [VP] * 7 + [I, VP]
    lib.hqq_b200_glue_moe_combine.argtypes = [VP] * 5 + [I] * 4 + [VP]
    lib.hqq_b200_linear_fwd_grouped.argtypes = [VP, VP, I, VP, VP, VP, VP, VP, I64, I, VP, VP, I64, I, I, I, VP]
    return lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def run_route(emu, x, router, k, ticket=None):
    M, H = x.shape
    E = router.shape[0]
    out = {"ids": torch.full((M, k), -7, dtype=torch.int32), "w": torch.full((M, k), float("nan")),
           "pair_of": torch.full((M, k), -7, dtype=torch.int32), "off": torch.full((E,), -7, dtype=torch.int32),
           "cnt": torch.full((E,), -7, dtype=torch.int32), "token": torch.full((M * k,), -7, dtype=torch.int32)}
    ticket = torch.zeros(1, dtype=torch.int32) if ticket is None else ticket
    rc = emu.hqq_b200_glue_moe_route(P(x), P(router), M, H, E, k, P(out["ids"]), P(out["w"]), P(out["pair_of"]), P(out["off"]), P(out["cnt"]),
                                     P(out["token"]), P(ticket), CODE[x.dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    assert int(ticket[0]) == 0, "the router must leave its ticket at zero"
    return out


def check_grouping(out, E):
    """The grouping is a function of the id table: compare with the restatement built from the kernel's own ids."""
    off, cnt, token, pair_of = MR.group(out["ids"], E)
    assert torch.equal(out["off"], off) and torch.equal(out["cnt"], cnt)
    assert torch.equal(out["token"], token) and torch.equal(out["pair_of"], pair_of)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("E,k", [(8, 1), (8, 2), (64, 4)])
@pytest.mark.parametrize("M", [1, 3, 33, 300])
def test_router_matches_the_restatement(emu, M, E, k, dtype):
    g = torch.Generator().manual_seed(M * 131 + E * 7 + k)
    H = 128
    x = torch.randn(M, H, generator=g).to(dtype)
    router = (torch.randn(E, H, generator=g) * 0.5).to(dtype)
    out = run_route(emu, x, router, k)
    ids, w, p = MR.route(x, router, k)
    tie = MR.near_tie(p, k)
    assert int(tie.sum()) <= max(1, M // 20), "too many near-ties for the comparison to mean anything"
    keep = ~tie
    assert torch.equal(out["ids"][keep], ids[keep])
    torch.testing.assert_close(out["w"][keep], w[keep], rtol=2e-6, atol=1e-7)
    assert torch.isfinite(out["w"]).all() and bool(((out["ids"] >= 0) & (out["ids"] < E)).all())
    check_grouping(out, E)


def test_router_exact_ties_go_to_the_lower_index(emu):
    H, E, k = 64, 8, 2
    x = torch.ones(3, H, dtype=torch.float16)
    router = torch.zeros(E, H, dtype=torch.float16)
    router[5] = 0.01  # experts 2 and 5 tie at the top, 1 and 6 tie behind them
    router[2] = 0.01
    router[1] = 0.005
    router[6] = 0.005
    out = run_route(emu, x, router, k)
    assert out["ids"].tolist() == [[2, 5]] * 3
    assert torch.equal(out["w"], torch.full((3, 2), 0.5))
    out1 = run_route(emu, x, router, 1)
    assert out1["ids"].tolist() == [[2]] * 3
    out3 = run_route(emu, x, router, 3)
    assert out3["ids"].tolist() == [[2, 5, 1]] * 3


def test_router_groups_many_rows_onto_one_expert(emu):
    """Every row routed to experts 3 and 6: groups of 40 pairs (more than one 32-row chunk), six experts without rows, tokens in
    ascending order within an expert."""
    M, H, E, k = 40, 64, 8, 2
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(M, H, generator=g) + 0.5).to(torch.float16)
    router = torch.zeros(E, H, dtype=torch.float16)
    router[3] = 0.05
    router[6] = 0.04
    out = run_route(emu, x, router, k)
    assert out["ids"].tolist() == [[3, 6]] * M
    assert out["cnt"].tolist() == [0, 0, 0, M, 0, 0, M, 0]
    assert out["off"].tolist() == [0, 0, 0, 0, M, M, M, 2 * M]
    assert out["token"].tolist() == list(range(M)) * 2
    assert out["pair_of"][:, 0].tolist() == list(range(M)) and out["pair_of"][:, 1].tolist() == list(range(M, 2 * M))
    check_grouping(out, E)


def test_router_rejects_bad_arguments(emu):
    H = 64
    x = torch.zeros(4, H, dtype=torch.float16)
    r = torch.zeros(64, H, dtype=torch.float16)
    b = [torch.zeros(4096, dtype=torch.int32) for _ in range(6)]
    t = torch.zeros(1, dtype=torch.int32)

    def call(M=4, E=8, k=2, xx=x, rr=r, ticket=t, Hh=H):
        return emu.hqq_b200_glue_moe_route(P(xx), P(rr), M, Hh, E, k, *[P(v) for v in b], P(ticket), F16, None)
    assert call() == 0
    for kw in ({"E": 1}, {"E": 65}, {"k": 0}, {"k": 9}, {"E": 4, "k": 5}, {"M": 0}, {"M": 65536}, {"Hh": 60}, {"xx": None}, {"rr": None},
               {"ticket": None}):
        assert call(**kw) == E_INVALID, kw
    assert emu.hqq_b200_glue_moe_route(P(x), P(r), 4, H, 8, 2, P(b[0]), None, *[P(v) for v in b[2:]], P(t), F16, None) == E_INVALID


# ---- expert-grouped forward ----------------------------------------------------------------------------------------------------
def draw_experts(seed, E, N, K, nbits, gs, dtype):
    g = FR.generator(seed, "cpu")
    layers = [FR.draw_layer(g, N, K, nbits, gs, dtype) for _ in range(E)]
    stack = lambda f: torch.stack([f(L) for L in layers]).contiguous()
    return layers, stack(lambda L: L.W_q), stack(lambda L: L.s.reshape(-1)), stack(lambda L: L.z.reshape(-1))


def run_grouped(emu, x, tables, mats, K, E, max_pairs, rows_out, gs, nbits, dtype, x_rows=True):
    """mats: [(W_q stack, scale stack, zero stack, N)]; returns the outputs [rows_out, N] (0x7BBB-filled before the launch)."""
    off, cnt, token = tables
    n = len(mats)
    ys = [torch.full((rows_out, N), 0x7BBB, dtype=torch.int16).view(dtype) for (_, _, _, N) in mats]
    arr = lambda ts: (VP * n)(*[t.data_ptr() for t in ts])
    rc = emu.hqq_b200_linear_fwd_grouped(P(x), P(token) if x_rows else None, n, arr([m[0] for m in mats]), arr([m[1] for m in mats]),
                                         arr([m[2] for m in mats]), arr(ys), (I64 * n)(*[m[3] for m in mats]), K, E, P(off), P(cnt), max_pairs,
                                         gs, nbits, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    return ys


def random_ids(g, M, E, k, skew=None):
    """[M, k] distinct experts per row; skew e: every row's first expert is e."""
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(M)]).to(torch.int32)
    if skew is not None:
        for t in range(M):
            row = ids[t].tolist()
            if skew in row:
                row.remove(skew)
            ids[t] = torch.tensor([skew] + row[:k - 1], dtype=torch.int32)
    return ids


@pytest.mark.parametrize("nbits,gs,dtype", [(4, 64, torch.float16), (2, 128, torch.bfloat16)])
@pytest.mark.parametrize("M,k,skew", [(1, 2, None), (3, 2, None), (20, 2, 5)])
def test_grouped_forward_matches_float64(emu, nbits, gs, dtype, M, k, skew):
    E, K, N, N2 = 8, 512, 256, 128
    layers, Wq, s, z = draw_experts(11 + M, E, N, K, nbits, gs, dtype)
    layers2, Wq2, s2, z2 = draw_experts(12 + M, E, N2, K, nbits, gs, dtype)
    g = torch.Generator().manual_seed(M)
    ids = random_ids(g, M, E, k, skew)
    off, cnt, token, _ = MR.group(ids, E)
    x = FR.draw_x(FR.generator(3, "cpu"), M, K, gs, dtype)
    P_ = M * k
    y, y2 = run_grouped(emu, x, (off, cnt, token), [(Wq, s, z, N), (Wq2, s2, z2, N2)], K, E, P_, P_ + 3, gs, nbits, dtype)
    for e in range(E):
        a, c = int(off[e]), int(cnt[e])
        if c == 0:
            continue
        xr = x[token[a:a + c].long()]
        FR.check(y[a:a + c], FR.reference(layers[e], xr, 1), f"gate expert {e}")
        FR.check(y2[a:a + c], FR.reference(layers2[e], xr, 1), f"up expert {e}")
    sentinel = torch.full((3, N), 0x7BBB, dtype=torch.int16)
    assert torch.equal(y[P_:].view(torch.int16), sentinel), "rows no pair owns must stay untouched"


def test_grouped_forward_rows_are_independent(emu):
    """Permuting the tokens and adding rows under the same max_pairs leaves every (token, expert) output's bits unchanged; x rows
    taken in pair order (x_rows NULL, the down projection) give the same bits as the gather."""
    E, K, N, nbits, gs, dtype, k = 8, 512, 256, 4, 64, torch.float16, 2
    _, Wq, s, z = draw_experts(21, E, N, K, nbits, gs, dtype)
    g = torch.Generator().manual_seed(9)
    M = 12
    ids = random_ids(g, M, E, k, skew=1)
    x = FR.draw_x(FR.generator(4, "cpu"), M, K, gs, dtype)
    max_pairs = 40
    off, cnt, token, pair_of = MR.group(ids, E)
    (y,) = run_grouped(emu, x, (off, cnt, token), [(Wq, s, z, N)], K, E, max_pairs, max_pairs, gs, nbits, dtype)
    perm = torch.randperm(M, generator=g)
    extra = 7
    ids2 = torch.cat([ids[perm], random_ids(g, extra, E, k)])
    x2 = torch.cat([x[perm], FR.draw_x(FR.generator(5, "cpu"), extra, K, gs, dtype)])
    off2, cnt2, token2, pair_of2 = MR.group(ids2, E)
    (y2,) = run_grouped(emu, x2, (off2, cnt2, token2), [(Wq, s, z, N)], K, E, max_pairs, max_pairs, gs, nbits, dtype)
    for i, t in enumerate(perm.tolist()):
        for j in range(k):
            a, b = int(pair_of[t, j]), int(pair_of2[i, j])
            assert torch.equal(y[a].view(torch.int16), y2[b].view(torch.int16)), (t, j)
    xg = x[token.long()].contiguous()  # rows already in pair order
    (y3,) = run_grouped(emu, xg, (off, cnt, token), [(Wq, s, z, N)], K, E, max_pairs, max_pairs, gs, nbits, dtype, x_rows=False)
    assert torch.equal(y3[:M * k].view(torch.int16), y[:M * k].view(torch.int16))


def test_grouped_forward_rejects_bad_arguments(emu):
    E, K, N = 8, 512, 256
    _, Wq, s, z = draw_experts(1, E, N, K, 4, 64, torch.float16)
    x = torch.zeros(4, K, dtype=torch.float16)
    tab = torch.zeros(E, dtype=torch.int32)
    y = torch.zeros(8, N, dtype=torch.float16)
    one = lambda t: (VP * 1)(t.data_ptr())

    def call(E=E, mp=8, nb=4, gs=64, dt=F16, off=tab, K=K):
        return emu.hqq_b200_linear_fwd_grouped(P(x), None, 1, one(Wq), one(s), one(z), one(y), (I64 * 1)(N), K, E, P(off), P(tab), mp, gs, nb,
                                               dt, None)
    assert call() == 0
    for kw in ({"E": 0}, {"E": 65}, {"mp": 0}, {"mp": 65535 * 8 + 1}, {"off": None}):
        assert call(**kw) == E_INVALID, kw
    for kw in ({"gs": 32}, {"nb": 8, "dt": BF16}, {"K": 384}):
        assert call(**kw) == E_UNSUPPORTED, kw


# ---- combine ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("k", [1, 2, 4])
def test_combine_is_bit_exact(emu, k, dtype):
    E, M, H = 8, 9, 96
    g = torch.Generator().manual_seed(k)
    ids = random_ids(g, M, E, k)
    w = torch.softmax(torch.randn(M, k, generator=g), dim=-1)
    _, _, _, pair_of = MR.group(ids, E)
    y = (torch.randn(M * k, H, generator=g) * 3).to(dtype)
    delta = torch.full((M, H), 7.0, dtype=dtype)
    rc = emu.hqq_b200_glue_moe_combine(P(y), P(ids), P(w), P(pair_of), P(delta), M, H, k, CODE[dtype], None)
    assert rc == 0, emu.hqq_b200_last_error()
    ref = MR.combine(y, ids, w, pair_of, E)
    assert torch.equal(delta.view(torch.int16), ref.view(torch.int16))
    assert emu.hqq_b200_glue_moe_combine(P(y), P(ids), P(w), None, P(delta), M, H, k, CODE[dtype], None) == E_INVALID
    assert emu.hqq_b200_glue_moe_combine(P(y), P(ids), P(w), P(pair_of), P(delta), M, H, 9, CODE[dtype], None) == E_INVALID


# ---- the harness's checks ------------------------------------------------------------------------------------------------------
def test_moe_shape_checks_raise_without_a_gpu():
    from hqq_b200.harness import MIXTRAL_8X7B, DecodeModel, LlamaShape
    assert MIXTRAL_8X7B.n_experts == 8 and MIXTRAL_8X7B.experts_per_token == 2 and MIXTRAL_8X7B.vocab == 32000
    assert LlamaShape().n_experts == 0
    small = dict(hidden=256, inter=512, n_layers=1, n_heads=2, n_kv_heads=1, vocab=64)
    for bad in ({"n_experts": 1}, {"n_experts": 65}, {"n_experts": 8, "experts_per_token": 0}, {"n_experts": 8, "experts_per_token": 9},
                {"n_experts": 4, "experts_per_token": 5}, {"n_experts": 16, "experts_per_token": 9}):
        with pytest.raises(ValueError):
            LlamaShape(**small, **bad)
    LlamaShape(**small, n_experts=64, experts_per_token=8)
    with pytest.raises(ValueError, match="tp"):
        DecodeModel(LlamaShape(**small, n_experts=8), device="meta", tp=2)
