"""CPU: the element-wise checks of tests/test_fused_forward_exact_gpu.py on the kernel emulator (tests/emu), fp16 and bf16, and
checks of tests/fused_ref.py itself.

The one-token and generic small-M kernels of csrc/linear_small.cu run their own source on the emulator at ragged N with several row
tiles per CTA; every output element must lie within fused_ref's bound of the float64 reference, and the bound must reject the
negative controls.  fused_ref's bound is also held against a float32 simulation of the route-1 arithmetic written out here in
numpy, so a bound that the kernel's own operation order could exceed is caught without a GPU."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import fused_ref as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
import run_small as RS  # noqa: E402

DT = {"float16": torch.float16, "bfloat16": torch.bfloat16}


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    return lib


def route_of(lib, M, L):
    return lib.hqq_b200_linear_fwd_route(ctypes.c_int64(M), ctypes.c_int64(L.N), ctypes.c_int64(L.K), L.gs, L.nbits, 1, RS.code_of(L.dtype))


def verify(y, ref, what):
    worst = F.check(y, ref, what)
    F.assert_controls_rejected(ref, what)
    return worst


@pytest.mark.parametrize("dt,nbits,gs,K,off", RS.EXACT_ONE_TOKEN)
def test_emulated_one_token_kernel_is_exact(emu, dt, nbits, gs, K, off):
    N = (8 // nbits) * RS.EXACT_STEP
    gen = F.generator(K + 10 * nbits + gs + off, "cpu")
    L = F.draw_layer(gen, N, K, nbits, gs, DT[dt], bias=(K % 512 == 0))
    x = F.draw_x(gen, 1, K, gs, DT[dt])
    assert route_of(emu, 1, L) == 1
    y = RS.linear_fwd(emu, x, L, meta_offset=off)
    verify(y, F.reference(L, x, 1), f"{dt} {nbits}b gs{gs} K{K} meta+{off}")


@pytest.mark.parametrize("dt,nbits,gs,K,M", RS.EXACT_SMALL_M)
def test_emulated_small_m_kernel_is_exact(emu, dt, nbits, gs, K, M):
    N = (8 // nbits) * RS.EXACT_STEP
    gen = F.generator(1000 + M + 10 * nbits + gs, "cpu")
    L = F.draw_layer(gen, N, K, nbits, gs, DT[dt], bias=(M % 2 == 1))
    x = F.draw_x(gen, M, K, gs, DT[dt])
    assert route_of(emu, M, L) == 1
    y = RS.linear_fwd(emu, x, L)
    verify(y, F.reference(L, x, 1), f"{dt} {nbits}b gs{gs} K{K} M{M}")


@pytest.mark.parametrize("dt,nbits,K", RS.EXACT_DECODE)
def test_emulated_prologues_and_paired_epilogue_are_exact(emu, dt, nbits, K):
    """x_op 1 with and without x2 (h_out == T(x + x2) bit for bit), x_op 2, and the paired SiLU * mul epilogue, which must equal
    T(T(silu(g)) * u) of the kernel's own g and u (the emulator's exp is expf) and lie within the propagated bound."""
    T = DT[dt]
    N = (8 // nbits) * RS.EXACT_STEP
    gen = F.generator(2000 + K + nbits, "cpu")
    La, Lb = F.draw_layer(gen, N, K, nbits, 64, T), F.draw_layer(gen, N, K, nbits, 64, T)
    x = F.on_grid(F.draw_x(gen, 1, K, 64, T), T)  # multiples of 1/16: the kernel's fp32 sum of squares is exact
    x2 = F.on_grid(F.draw_x2(gen, K, 64, T), T)
    w = (torch.rand(K, generator=gen) + 0.5).to(T)
    for tag, xop, with_x2 in (("rmsnorm+x2", 1, True), ("rmsnorm", 1, False), ("silu*mul", 2, True)):
        if xop == 1:
            h_ref, act, slack = F.prologue_rmsnorm(x, x2 if with_x2 else None, w, 1e-5, T)
        else:
            act, slack = F.prologue_silu_mul(x, x2, T)
        xs = dict(x2=x2 if with_x2 else None, xw=w if xop == 1 else None, want_h=(xop == 1))
        (ya, yb), h = RS.decode_linear_fwd(emu, x, [La, Lb], xop, **xs)
        if xop == 1:
            assert torch.equal(h, h_ref), tag
        ra, rb = F.reference(La, act, 1, x_slack=slack), F.reference(Lb, act, 1, x_slack=slack)
        verify(ya, ra, f"{tag} (a)")
        verify(yb, rb, f"{tag} (b)")
        (act_p, _), h2 = RS.decode_linear_fwd(emu, x, [La, Lb], xop | 16, **xs)
        restated = (F.silu_f32(ya).to(T).float() * yb.float()).to(T)
        assert torch.equal(act_p, restated), f"paired {tag}"
        bnd, exact = F.silu_mul_bound(ra, rb)
        assert bool(((act_p.to(torch.float64) - exact).abs() <= bnd).all()), f"paired {tag}"
        if xop == 1:
            assert torch.equal(h2, h_ref), tag


# ------------------------------------------------------------------------------------------------------------- fused_ref itself
def _f32(v):
    return np.float32(v) if np.isscalar(v) else np.asarray(v, dtype=np.float32)


def _fma(a, b, c):
    """fp32 fma: the float64 product of two float32 values is exact, one rounding of the sum to float32 (the float64 sum may round
    first; at these magnitudes that never matters for a bound check)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def simulate_route1(L, x):
    """numpy float32 restatement of linear_decode1_kernel / linear_small_kernel for token 0: per group, the planted lanes OFF + q
    contracted with x (fp32, k by k), the group sum of x, tot = fma(s, S, fma(-s (OFF + z), X, tot)) per warp over its chunk of
    256-k units, the eight warp partials added in warp order, T(.) and + bias in T."""
    N, K, gs = L.N, L.K, L.gs
    off = F.OFF[L.dtype]
    q = L.q.reshape(N, K).numpy().astype(np.float32)
    s = L.s.reshape(N, K // gs).to(torch.float32).numpy()
    z = L.z.reshape(N, K // gs).to(torch.float32).numpy()
    xv = x[0].to(torch.float32).numpy()
    KB = K // 256
    parts = []
    for w in range(8):
        tot = np.zeros(N, dtype=np.float32)
        for g in range(KB * w // 8 * 256 // gs, KB * (w + 1) // 8 * 256 // gs):
            S = np.zeros(N, dtype=np.float32)
            X = np.float32(0)
            for k in range(g * gs, (g + 1) * gs):
                S = (S + (off + q[:, k]) * xv[k]).astype(np.float32)
                X = np.float32(X + xv[k])
            tot = _fma(s[:, g], S, _fma(_f32(-s[:, g] * _f32(off + z[:, g])), np.full(N, X, np.float32), tot))
        parts.append(tot)
    acc = np.zeros(N, dtype=np.float32)
    for p in parts:
        acc = (acc + p).astype(np.float32)
    y = torch.from_numpy(acc).to(L.dtype)[None]
    return y if L.bias is None else y + L.bias


@pytest.mark.parametrize("dt", ["float16", "bfloat16"])
@pytest.mark.parametrize("nbits,gs,K", [(4, 64, 2304), (1, 128, 768), (2, 64, 4352)])
def test_fused_ref_bound_holds_for_a_float32_simulation_and_rejects_the_controls(dt, nbits, gs, K):
    gen = F.generator(nbits * 100 + K, "cpu")
    L = F.draw_layer(gen, 16 * (8 // nbits), K, nbits, gs, DT[dt], bias=True)
    x = F.draw_x(gen, 1, K, gs, DT[dt])
    ref = F.reference(L, x, 1)
    worst = F.check(simulate_route1(L, x), ref, "simulation")
    assert worst < 1.0
    assert F.assert_controls_rejected(ref) > 1.0
    # routes 2 and 3: fp32 k-by-k accumulation of x * W_r, the reference's two roundings in W_r
    W_r = L.dequantized().to(torch.float32)
    acc = torch.zeros(L.N, dtype=torch.float32)
    for k in range(K):
        acc = acc + x[0, k].to(torch.float32) * W_r[:, k]
    y2 = acc.to(L.dtype)[None] + L.bias
    ref2 = F.reference(L, x, 2)
    F.check(y2, ref2, "route-2 simulation")
    F.assert_controls_rejected(ref2)


def test_fused_ref_rounding_helpers():
    v = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, 2 ** -20, -65504.0, 0.1, 3.0e-8], dtype=torch.float64)
    assert np.array_equal(F.round_to(v, torch.float16).numpy(), v.numpy().astype(np.float16))  # numpy: one correct rounding
    assert torch.equal(F.ulp(torch.tensor([1.0, 1.5, 2.0, 2 ** -30]), torch.float16), torch.tensor([2 ** -10, 2 ** -10, 2 ** -9, 2 ** -24],
                                                                                                   dtype=torch.float64))
    assert float(F.ulp(torch.tensor([1.0]), torch.bfloat16)) == 2 ** -7
    # a tie between two bf16 values rounds to even, a hair above rounds up
    assert float(F.round_to(torch.tensor([1.0 + 2 ** -8], dtype=torch.float64), torch.bfloat16)) == 1.0
    assert float(F.round_to(torch.tensor([1.0 + 2 ** -8 + 2 ** -30], dtype=torch.float64), torch.bfloat16)) == 1.0 + 2 ** -7
    assert math.isclose(F.route_d(1, 2304, 64), 64 // 16 + 5 + 12)
