"""GPU: the fused forward kernels element by element against a float64 reference of the same operation (tests/fused_ref.py), at the
shapes where their schedules change: several row tiles per CTA, long K, the one-token kernel's limits, ragged and uneven k-chunks,
the decode prologues and the paired epilogue, split-K with a short last slice, and both sides of the route boundaries.

Every case states the route it means to exercise (ops.linear_route), checks |y - y*| <= bound for EVERY output element, and checks
that the same comparison rejects three defects built from the same data (fused_ref.negative_controls).  A relative L2 norm over
the whole output would let one wrong row of a 4096-row layer through; these checks do not.

Instantiations reached (hqq_b200/csrc/linear_small.cu `sk_mt`, linear_gemm.cu `by_bits`), per dtype, width and group size the routers
accept:
  one-token ST = 2 (8-bit, fp16)               test_one_token_kernel (nbits 8)
  one-token ST = 4, MR = 0 (register meta)     test_one_token_kernel (K % 512 != 0, gs 128, 8-byte-offset meta), test_long_k
  one-token ST = 4, MR = 1 (meta on the ring)  test_one_token_kernel (gs 64, K = 2048), test_long_k (gs 64)
  small-M MT = 1 / 2 / 4                        test_small_m_kernel (M = 2, 8 / 9, 16 / 17, 32), test_long_k (M = 1, K > 16384)
  wgmma GEMM, every width and group size       test_gemm_full_size, test_gemm_8bit_bf16_few_tokens
  dequantize + dense wgmma GEMM                 test_route3

The largest err / bound of every case is printed (run with -s to see it)."""
import math

import pytest
import torch

import fused_ref as R
from hqq_b200 import ops
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr
from hqq_b200.core.quantize import HQQLinear, Quantizer

pytestmark = pytest.mark.gpu
DEV = "cuda"
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
WIDTHS = [("f16", 8), ("f16", 4), ("f16", 2), ("f16", 1), ("bf16", 4), ("bf16", 2), ("bf16", 1)]  # what route 1 accepts
N_MULTI = 4360  # 273 row tiles at every width: more than the 264 CTAs of one wave, so some CTAs run two tiles; ragged last tile


def hqq_layer(L):
    layer = HQQLinear(None, None, compute_dtype=L.dtype, device=DEV, initialize=False)
    pk = Quantizer.bit_to_packing[L.nbits]
    layer.W_q = torch.nn.Parameter(L.W_q, requires_grad=False)
    layer.meta = {"nbits": L.nbits, "group_size": L.gs, "shape": torch.Size((L.N, L.K)), "axis": L.axis, "packing": pk, "view_as_float": False,
                  "unpack_view_dtype": Quantizer.unpack_view_dtype[pk], "compute_dtype": L.dtype, "quant_scale": False, "quant_zero": False,
                  "scale": L.s, "zero": L.z}
    layer.bias = L.bias
    layer.ready = True
    layer.in_features, layer.out_features = L.K, L.N
    return layer


def offset_meta(layer):
    """The same scale / zero values 8 bytes past a 16-byte boundary: the one-token kernel must take its register meta path."""
    for name in ("scale", "zero"):
        t = layer.meta[name]
        buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=DEV)
        buf[4:].copy_(t.reshape(-1))
        layer.meta[name] = buf[4:].view(t.shape)
    assert layer.meta["scale"].data_ptr() % 16 == 8 and layer.meta["zero"].data_ptr() % 16 == 8


def draw(seed, N, K, nbits, gs, dt, axis=1, bias=False):
    gen = R.generator(seed, DEV)
    return gen, R.draw_layer(gen, N, K, nbits, gs, DT[dt], axis=axis, bias=bias, pack=ops.pack)


def verify(y, ref, what):
    """Every element within its bound, every negative control rejected; prints the case's largest err / bound."""
    torch.cuda.synchronize()
    worst = R.check(y, ref, what)
    R.assert_controls_rejected(ref, what)
    print(f"[fused-exact] {what}: max err/bound = {worst:.4f}")
    return worst


def run_route(layer, x, route):
    L_meta = layer.meta
    nb = Quantizer._packing_bits[L_meta["packing"]]
    M = x.shape[0]
    N, K = L_meta["shape"]
    assert ops.linear_route(M, N, K, L_meta["group_size"], nb, L_meta["axis"], x.dtype) == route, (M, N, K, route)
    return layer(x)


# ------------------------------------------------------------------------------------------------------------ 1. one-token kernel
@pytest.mark.parametrize("dt,nbits", WIDTHS)
@pytest.mark.parametrize("gs", [64, 128])
def test_one_token_kernel(dt, nbits, gs):
    """M = 1 at K = 256 / 768 / 2304 (1, 3 and 9 k-units: idle warps, uneven warp chunks, K % 512 != 0 -> register meta) and 2048
    (gs 64: meta on the ring), N = 4360 (273 tiles, two per CTA for some), bias on every other K; at gs 64 with K % 512 == 0 also the
    8-byte-offset meta view (register path), which must give the same bits."""
    for i, K in enumerate((256, 768, 2048, 2304)):
        gen, L = draw(1000 * nbits + 10 * gs + i, N_MULTI, K, nbits, gs, dt, bias=(i % 2 == 1))
        x = R.draw_x(gen, 1, K, gs, DT[dt])
        layer = hqq_layer(L)
        y = run_route(layer, x, 1)
        ref = R.reference(L, x, 1)
        verify(y, ref, f"one-token {dt} {nbits}b gs{gs} K{K}")
        if gs == 64 and K % 512 == 0 and nbits != 8:
            offset_meta(layer)
            y2 = run_route(layer, x, 1)
            verify(y2, ref, f"one-token {dt} {nbits}b gs{gs} K{K} register-meta")
            assert torch.equal(y, y2)


# ------------------------------------------------------------------------------------------------------------------ 2. long K
@pytest.mark.parametrize("dt,nbits", WIDTHS)
def test_long_k_one_token(dt, nbits):
    """gs 64, N = 4096, K = 14336 and 16384 (the one-token kernel's largest shared-memory footprint, 1 CTA/SM on the ring path, so
    CTAs run several tiles), ring and register meta paths."""
    for K in (14336, 16384):
        gen, L = draw(7 * nbits + K, 4096, K, nbits, 64, dt)
        x = R.draw_x(gen, 1, K, 64, DT[dt])
        layer = hqq_layer(L)
        y = run_route(layer, x, 1)
        ref = R.reference(L, x, 1)
        verify(y, ref, f"long-K {dt} {nbits}b K{K}")
        if nbits != 8:
            offset_meta(layer)
            y2 = run_route(layer, x, 1)
            verify(y2, ref, f"long-K {dt} {nbits}b K{K} register-meta")


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("K", [16640, 28672])
def test_long_k_generic_kernel(dt, K):
    """M = 1 past the one-token kernel's limit (K > 16384): the generic small-M kernel with MT = 1, 4-bit gs 64, N = 8192."""
    gen, L = draw(K + len(dt), 8192, K, 4, 64, dt, bias=True)
    x = R.draw_x(gen, 1, K, 64, DT[dt])
    y = run_route(hqq_layer(L), x, 1)
    verify(y, R.reference(L, x, 1), f"generic M=1 {dt} K{K}")


# -------------------------------------------------------------------------------------------------------------- 3. small-M kernel
@pytest.mark.parametrize("dt,nbits", WIDTHS)
@pytest.mark.parametrize("gs", [64, 128])
def test_small_m_kernel(dt, nbits, gs):
    """The generic kernel at M = 2, 8 (MT 1), 9, 16 (MT 2), 17, 32 (MT 4), K = 2304 (9 units: uneven chunks), N = 4360."""
    K = 2304
    gen, L = draw(3000 + 10 * nbits + gs + len(dt), N_MULTI, K, nbits, gs, dt, bias=True)
    layer = hqq_layer(L)
    for M in (2, 8, 9, 16, 17, 32):
        x = R.draw_x(gen, M, K, gs, DT[dt])
        y = run_route(layer, x, 1)
        verify(y, R.reference(L, x, 1), f"small-M {dt} {nbits}b gs{gs} M{M}")


@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_route_boundary_17_to_32_tokens(dt):
    """N K = 2^24 is the last size route 1 takes at 17 <= M <= 32: (4096, 4096) runs the small-M kernel, (4096, 4352) the wgmma GEMM."""
    for (N, K), route in (((4096, 4096), 1), ((4096, 4352), 2)):
        gen, L = draw(N + K, N, K, 4, 64, dt)
        layer = hqq_layer(L)
        for M in (17, 32):
            x = R.draw_x(gen, M, K, 64, DT[dt])
            y = run_route(layer, x, route)
            ks = ksplit_of(M, N, K, 64, 4, DT[dt]) if route == 2 else 1
            if route == 2:
                assert torch.equal(layer.dequantize(), L.dequantized())
            verify(y, R.reference(L, x, route, ksplit=ks), f"boundary {dt} N{N} K{K} M{M} route {route}")


# --------------------------------------------------------------------------------------------------- 4. prologues / paired epilogue
def glue_silu_mul(g, u):
    out = torch.empty_like(g)
    check(load().hqq_b200_glue_silu_mul(ptr(g), ptr(u), ptr(out), g.numel(), DTYPE_CODE[g.dtype], stream_ptr(g.device)))
    return out


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("nbits", [4, 2])
@pytest.mark.parametrize("K", [256, 2304, 5120, 14336, 16384])
def test_decode_prologues_and_paired_epilogue(dt, nbits, K):
    """ops.decode_linear_fwd with x_op 1 (residual add + RMSNorm, with and without x2; h_out must be T(x + x2) bit for bit), x_op 2
    (SiLU * mul) and x_op | YOP_SILU_MUL_PAIR.  K = 5120 leaves a partial second staging vector (K % 4096 != 0); K >= 5120 gives
    warps chunks over 512 elements (norm weights loaded inside the loop).  The reference activation follows the documented
    roundings; the bound is widened by the activation's possible last-ulp flips."""
    T = DT[dt]
    N = 2056
    gen = R.generator(5000 + K + nbits + len(dt), DEV)
    La = R.draw_layer(gen, N, K, nbits, 64, T, pack=ops.pack)
    Lb = R.draw_layer(gen, N, K, nbits, 64, T, pack=ops.pack)
    A, B = hqq_layer(La), hqq_layer(Lb)
    x = R.on_grid(R.draw_x(gen, 1, K, 64, T), T)  # multiples of 1/16: the kernel's fp32 sum of squares is exact
    x2 = R.on_grid(R.draw_x2(gen, K, 64, T), T)
    w = (torch.rand(K, generator=gen, device=DEV) + 0.5).to(T)
    eps = 1e-5
    for tag, xop, with_x2 in (("rmsnorm+x2", 1, True), ("rmsnorm", 1, False), ("silu*mul", 2, True)):
        if xop == 1:
            h_ref, act, slack = R.prologue_rmsnorm(x, x2 if with_x2 else None, w, eps, T)
        else:
            act, slack = R.prologue_silu_mul(x, x2, T)
        ya, yb = (torch.empty(1, N, device=DEV, dtype=T) for _ in range(2))
        h = torch.empty(1, K, device=DEV, dtype=T) if xop == 1 else None
        assert ops.decode_linear_fwd(x, (A, B), [ya, yb], xop, x2 if with_x2 else None, w if xop == 1 else None, h, eps)
        torch.cuda.synchronize()
        if xop == 1:
            assert torch.equal(h, h_ref), f"h_out {tag}"
        ra, rb = R.reference(La, act, 1, x_slack=slack), R.reference(Lb, act, 1, x_slack=slack)
        verify(ya, ra, f"prologue {tag} {dt} {nbits}b K{K} (a)")
        verify(yb, rb, f"prologue {tag} {dt} {nbits}b K{K} (b)")
        # the paired epilogue: y[0] = T(T(silu(g)) * u) from one launch, g and u the kernel's own products
        act_p, keep = torch.empty(1, N, device=DEV, dtype=T), torch.full((1, N), 7.0, device=DEV, dtype=T)
        assert ops.decode_linear_fwd(x, (A, B), [act_p, keep], xop | ops.YOP_SILU_MUL_PAIR, x2 if with_x2 else None, w if xop == 1 else None,
                                     None, eps)
        torch.cuda.synchronize()
        assert bool((keep == 7.0).all()), "the paired epilogue wrote y[1]"
        # the same roundings, and the same __expf, as the decode glue's silu_mul kernel
        assert torch.equal(act_p, glue_silu_mul(ya, yb)), f"paired {tag}: not T(T(silu(g)) * u) of the kernel's own g, u"
        bnd, exact = R.silu_mul_bound(ra, rb)
        err = (act_p.to(torch.float64) - exact).abs()
        assert bool((err <= bnd).all()), f"paired {tag}: max err/bound {float((err / bnd).max()):.3g}"
        print(f"[fused-exact] paired {tag} {dt} {nbits}b K{K}: max err/bound = {float((err / bnd).max()):.4f}")


# ------------------------------------------------------------------------------------------------------------ 5. route 2 full size
def ksplit_of(M, N, K, gs, nbits, dtype):
    """k-slices of the wgmma schedule, read off the split-K workspace it asks for ([ksplit][row tiles][token tiles][128][128] fp32)."""
    lib = load()
    ws = int(lib.hqq_b200_linear_fwd_workspace_bytes(M, N, K, gs, nbits, 1, DTYPE_CODE[dtype]))
    F = 8 // nbits
    tiles = math.ceil(N // F / (128 // F)) * math.ceil(M / 128)
    assert ws % (tiles * 128 * 128 * 4) == 0
    return max(1, ws // (tiles * 128 * 128 * 4))


GEMM_WIDTHS = [(dt, nb) for dt in ("f16", "bf16") for nb in (8, 4, 2, 1)]


@pytest.mark.parametrize("dt,nbits", GEMM_WIDTHS)
@pytest.mark.parametrize("gs", [64, 128])
def test_gemm_full_size(dt, nbits, gs):
    """Route 2 at (N, K, M) = (4096, 4096, 600) (several token tiles), (1024, 14336, 64) (split-K, 8 slices), (1024, 11008, 48) (43
    quads over 8 slices: the last slice gets one) and (14336, 4096, 33) (a 33rd token in a second tile)."""
    for i, (N, K, M) in enumerate(((4096, 4096, 600), (1024, 14336, 64), (1024, 11008, 48), (14336, 4096, 33))):
        gen, L = draw(7000 + 100 * nbits + gs + i + len(dt), N, K, nbits, gs, dt, bias=(i % 2 == 0))
        layer = hqq_layer(L)
        assert torch.equal(layer.dequantize(), L.dequantized())
        x = R.draw_x(gen, M, K, gs, DT[dt])
        y = run_route(layer, x, 2)
        ks = ksplit_of(M, N, K, gs, nbits, DT[dt])
        assert (ks > 1) == (N == 1024), (N, K, M, ks)  # few tiles: split-K; many: none
        verify(y, R.reference(L, x, 2, ksplit=ks), f"gemm {dt} {nbits}b gs{gs} N{N} K{K} M{M} ksplit {ks}")


def test_gemm_8bit_bf16_few_tokens():
    """8-bit bf16 never takes route 1: at M = 1..32 the wgmma GEMM runs one token tile with 96+ padded token columns."""
    for M in (1, 16, 32):
        gen, L = draw(9000 + M, 4096, 4096, 8, 64, "bf16", bias=True)
        layer = hqq_layer(L)
        x = R.draw_x(gen, M, 4096, 64, torch.bfloat16)
        y = run_route(layer, x, 2)
        ks = ksplit_of(M, 4096, 4096, 64, 8, torch.bfloat16)
        verify(y, R.reference(L, x, 2, ksplit=ks), f"gemm bf16 8b M{M} ksplit {ks}")


# -------------------------------------------------------------------------------------------------------------------- 6. route 3
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("nbits,axis", [(3, 1), (4, 0)])
def test_route3(dt, nbits, axis):
    """3-bit and axis 0: the dequantize kernel, then the dense wgmma GEMM, at (4096, 4096)."""
    gen, L = draw(11000 + 10 * nbits + axis + len(dt), 4096, 4096, nbits, 64, dt, axis=axis)
    layer = hqq_layer(L)
    assert torch.equal(layer.dequantize(), L.dequantized())
    for M in (1, 48):
        x = R.draw_x(gen, M, 4096, 64, DT[dt])
        y = run_route(layer, x, 3)
        verify(y, R.reference(L, x, 3), f"route3 {dt} {nbits}b axis{axis} M{M}")
