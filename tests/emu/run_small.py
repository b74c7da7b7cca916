"""TEST INFRASTRUCTURE ONLY: run the emulated small-M / one-token forward (csrc/linear_small.cu on the fiber emulator) over a fixed
seeded case list under the HQQ_B200_* knobs of THIS process and save every output to an .npz.  tests/test_emu_cpu.py compares the
default run with the oracle and the knob runs with the default run (the knobs are read once per process, hence one process each).
tests/test_fused_forward_exact_cpu.py calls `linear_fwd` / `decode_linear_fwd` below in its own process for the EXACT_* cases."""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import build_emu  # noqa: E402
from oracle import hqq_oracle as O  # noqa: E402

F16, BF16 = 1, 2


def P(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def aligned(shape, dtype, align=256):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.zeros(n + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + n].view(dtype).reshape(shape)


def dev(a, dtype=None):
    a = np.asarray(a, dtype=dtype)
    d = aligned(a.shape, a.dtype)
    d[...] = a
    return d


def make_layer(rng, N, K, nbits, gs, with_bias=False):
    R = N * K // gs
    levels = rng.integers(0, 2 ** nbits, size=(R, gs))
    Wq = O.PACK[O.BIT_TO_PACKING[nbits]](levels)
    scale = (rng.random((R, 1)) * 0.01 + 2e-3).astype(np.float16)
    zero = (rng.random((R, 1)) * (2 ** nbits - 1)).astype(np.float16)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float16) if with_bias else None
    meta = {"nbits": nbits, "group_size": gs, "shape": (N, K), "axis": 1, "packing": O.BIT_TO_PACKING[nbits],
            "scale": scale.astype(np.float32), "zero": zero.astype(np.float32)}
    return {"Wq": dev(Wq), "scale": dev(scale[:, 0]), "zero": dev(zero[:, 0]), "bias": None if bias is None else dev(bias), "meta": meta,
            "Wq_host": Wq, "bias_host": bias, "N": N, "K": K}


def dev_t(t, offset=0):
    """A CPU torch tensor as a 256-byte aligned numpy buffer (fp16 / bf16 as their 16-bit patterns), starting `offset` bytes past
    the boundary."""
    import torch
    a = t.contiguous()
    if a.dtype in (torch.float16, torch.bfloat16):
        a = a.view(torch.int16)
    a = a.numpy()
    if offset == 0:
        return dev(a)
    n = offset // a.itemsize
    buf = aligned((a.size + n,), a.dtype)
    buf[n:] = a.reshape(-1)
    return buf[n:].reshape(a.shape)


def _out(shape):
    return aligned(shape, np.uint16)  # 16-bit patterns of an fp16 / bf16 output, read back by _back


def _back(buf, dtype):
    import torch
    return torch.from_numpy(buf.copy().view(np.int16)).view(dtype)


def code_of(dtype):
    import torch
    return {torch.float16: F16, torch.bfloat16: BF16}[dtype]


def linear_fwd(lib, x, L, meta_offset=0):
    """hqq_b200_linear_fwd on the emulator for a fused_ref.Layer (route 1: no workspace) and an [M, K] activation in its dtype."""
    M, K = x.shape
    i64 = ctypes.c_int64
    bufs = [dev_t(x), dev_t(L.W_q), dev_t(L.s, meta_offset), dev_t(L.z, meta_offset), None if L.bias is None else dev_t(L.bias)]
    y = _out((M, L.N))
    rc = lib.hqq_b200_linear_fwd(*[P(b) for b in bufs], P(y), i64(M), i64(L.N), i64(K), L.gs, L.nbits, 1, code_of(L.dtype), None,
                                 ctypes.c_size_t(0), None)
    assert rc == 0, lib.hqq_b200_last_error()
    return _back(y, L.dtype)


def decode_linear_fwd(lib, x, layers, x_op, x2=None, xw=None, want_h=False, eps=1e-5):
    """hqq_b200_decode_linear_fwd on the emulator for fused_ref.Layers of equal N; returns (outputs, h_out or None)."""
    K, N, dt = x.shape[1], layers[0].N, layers[0].dtype
    n = len(layers)
    VP, i64 = ctypes.c_void_p, ctypes.c_int64
    keep = [dev_t(x)] + [None if t is None else dev_t(t) for t in (x2, xw)]
    mats = [(dev_t(L.W_q), dev_t(L.s), dev_t(L.z), None if L.bias is None else dev_t(L.bias)) for L in layers]
    ys = [_out((1, N)) for _ in layers]
    h = _out((1, K)) if want_h else None
    arr = lambda vals: (VP * n)(*[v.ctypes.data if v is not None else None for v in vals])  # noqa: E731
    rc = lib.hqq_b200_decode_linear_fwd(P(keep[0]), x_op, P(keep[1]), P(keep[2]), P(h), ctypes.c_float(eps), n, arr([m[0] for m in mats]),
                                        arr([m[1] for m in mats]), arr([m[2] for m in mats]), arr([m[3] for m in mats]), arr(ys),
                                        (i64 * n)(*[N] * n), i64(K), layers[0].gs, layers[0].nbits, code_of(dt), None)
    assert rc == 0, lib.hqq_b200_last_error()
    return [_back(y, dt) for y in ys], (None if h is None else _back(h, dt))


# (nbits, gs, N, K, M, bias)
PLAIN = [(4, 64, 32, 256, 1, False), (4, 64, 48, 512, 1, True), (4, 128, 32, 512, 1, False), (2, 64, 64, 256, 1, False), (1, 64, 64, 512, 1, True),
         (8, 64, 32, 256, 1, False), (4, 64, 40, 768, 1, False), (4, 64, 32, 2304, 1, False), (4, 64, 32, 1792, 1, False),
         (4, 64, 32, 256, 5, False), (2, 128, 64, 512, 3, True), (8, 64, 16, 256, 20, False), (4, 64, 48, 512, 32, False)]
# one-token kernel with prologues / paired epilogue: (nbits, N, K)
DECODE = [(4, 64, 512), (2, 64, 1024), (1, 128, 512), (4, 48, 1536), (4, 224, 512)]

# Element-wise cases of tests/test_fused_forward_exact_cpu.py (fp16 and bf16, fused_ref bounds).  N = F * EXACT_STEP: 211 packed rows
# make 14 / 27 / 53 / 106 row tiles at 8 / 4 / 2 / 1 bits, so every one of the emulator's 8 resident CTAs walks two or more tiles
# and the last tile is ragged.
EXACT_STEP = 211
# one-token kernel: (dtype, nbits, gs, K, scale/zero byte offset); K = 256 / 768 / 2304 are 1 / 3 / 9 k-units (idle warps, uneven
# chunks, register meta), K = 1024 at gs 64 takes the meta ring (offset 0) and the register meta (offset 8)
EXACT_ONE_TOKEN = [(dt, nb, gs, K, off) for dt in ("float16", "bfloat16") for nb in ((8, 4, 2, 1) if dt == "float16" else (4, 2, 1))
                   for gs, K, off in ((64, 256, 0), (128, 768, 0), (64, 1024, 0), (64, 1024, 8), (64, 2304, 0))]
# generic small-M kernel: (dtype, nbits, gs, K, M) -- MT = 1, 2, 4
EXACT_SMALL_M = [(dt, nb, gs, 768, M) for dt in ("float16", "bfloat16") for nb, gs in ((4, 64), (2, 128), (1, 64)) for M in (3, 9, 17)] + \
                [("float16", 8, 128, 768, 5), ("float16", 4, 64, 2304, 20)]
# one-token prologues and the paired epilogue: (dtype, nbits, K)
EXACT_DECODE = [(dt, nb, K) for dt in ("float16", "bfloat16") for nb in (4, 2) for K in (768, 2304)]


def main(out_path):
    lib = ctypes.CDLL(build_emu.build())
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    i64 = ctypes.c_int64
    res = {}
    for ci, (nbits, gs, N, K, M, wb) in enumerate(PLAIN):
        rng = np.random.default_rng(100 + ci)
        L = make_layer(rng, N, K, nbits, gs, wb)
        x = rng.standard_normal((M, K)).astype(np.float16)
        xd, y = dev(x), aligned((M, N), np.float16)
        rc = lib.hqq_b200_linear_fwd(P(xd), P(L["Wq"]), P(L["scale"]), P(L["zero"]), P(L["bias"]), P(y), i64(M), i64(N), i64(K), gs, nbits, 1, F16,
                                     None, ctypes.c_size_t(0), None)
        assert rc == 0, lib.hqq_b200_last_error()
        res[f"plain{ci}"] = y.copy()
        res[f"plain{ci}_ref"] = O.linear_forward(x.astype(np.float32), L["Wq_host"], L["meta"],
                                                 None if not wb else L["bias_host"].astype(np.float32), "float16")
    VP = ctypes.c_void_p
    for ci, (nbits, N, K) in enumerate(DECODE):
        rng = np.random.default_rng(200 + ci)
        A, B = make_layer(rng, N, K, nbits, 64), make_layer(rng, N, K, nbits, 64)
        x = rng.standard_normal((1, K)).astype(np.float16)
        x2 = (rng.standard_normal((1, K)) * 0.5).astype(np.float16)
        w = rng.random(K).astype(np.float16)
        xd, x2d, wd = dev(x), dev(x2), dev(w)
        arr = lambda vals: (VP * 2)(*[v.ctypes.data if v is not None else None for v in vals])  # noqa: E731
        Ns = (i64 * 2)(N, N)
        for tag, xop, use_x2, xw, want_h in (("x0", 0, False, None, False), ("x1", 1, True, wd, True), ("x2", 2, True, None, False),
                                             ("x1pair", 1 | 16, True, wd, True), ("x0pair", 16, False, None, False)):
            ya, yb = aligned((1, N), np.float16), aligned((1, N), np.float16)
            hout = aligned((1, K), np.float16) if want_h else None
            rc = lib.hqq_b200_decode_linear_fwd(P(xd), xop, P(x2d) if use_x2 else None, P(xw), P(hout), ctypes.c_float(1e-5), 2,
                                                arr([A["Wq"], B["Wq"]]), arr([A["scale"], B["scale"]]), arr([A["zero"], B["zero"]]),
                                                arr([None, None]), arr([ya, yb]), Ns, i64(K), 64, nbits, F16, None)
            assert rc == 0, lib.hqq_b200_last_error()
            res[f"dec{ci}_{tag}_a"] = ya.copy()
            if not (xop & 16):
                res[f"dec{ci}_{tag}_b"] = yb.copy()
            if want_h:
                res[f"dec{ci}_{tag}_h"] = hout.copy()
        # references for the plain one-token call
        for nm, Lr in (("a", A), ("b", B)):
            res[f"dec{ci}_x0_{nm}_ref"] = O.linear_forward(x.astype(np.float32), Lr["Wq_host"], Lr["meta"], None, "float16")
    np.savez(out_path, **res)


if __name__ == "__main__":
    main(sys.argv[1])
