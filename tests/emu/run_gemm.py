"""TEST INFRASTRUCTURE ONLY: run the emulated wgmma GEMM (csrc/linear_gemm.cu on the fiber emulator's functional model of
mbarrier / TMA / wgmma) over a fixed seeded case list under the HQQ_B200_* knobs of THIS process and save every output
plus the oracle's to an .npz (tests/test_emu_cpu.py compares)."""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import build_emu  # noqa: E402
import run_small as R  # noqa: E402
from oracle import hqq_oracle as O  # noqa: E402

# (nbits, gs, N, K, M, bias): ragged row tiles (N % 128 != 0), ragged token tiles, both UN (64/128), M > 256 and > 512 for the
# two-accumulator variant, few tiles x long K for split-K
CASES = [(4, 64, 128, 256, 64, False), (4, 64, 256, 512, 200, True), (2, 128, 128, 256, 40, False), (8, 64, 128, 256, 300, False),
         (1, 64, 256, 256, 64, True), (4, 64, 200, 512, 600, False), (4, 128, 136, 1024, 257, True), (2, 64, 64, 768, 1030, False),
         (4, 64, 128, 2048, 128, False), (4, 64, 264, 1280, 100, True), (8, 128, 128, 512, 513, False), (4, 64, 128, 256, 33, False)]


# route 3 (dequantize kernel -> dense wgmma GEMM, both operands on TMA): 3-bit, a group size the fused kernels do not take, ragged K
DENSE_CASES = [(3, 64, 130, 256, 40, True), (3, 64, 128, 512, 300, False), (4, 32, 128, 256, 64, False), (4, 64, 96, 320, 70, True),
               (2, 16, 64, 80, 33, False)]


def main(out_path):
    lib = ctypes.CDLL(build_emu.build())
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    lib.hqq_b200_linear_fwd_workspace_bytes.restype = ctypes.c_size_t
    lib.hqq_b200_linear_fwd_workspace_bytes.argtypes = [ctypes.c_int64] * 3 + [ctypes.c_int] * 4
    i64 = ctypes.c_int64
    res = {}
    for ci, (nbits, gs, N, K, M, wb) in enumerate(CASES):
        rng = np.random.default_rng(300 + ci)
        L = R.make_layer(rng, N, K, nbits, gs, wb)
        x = rng.standard_normal((M, K)).astype(np.float16)
        xd, y = R.dev(x), R.aligned((M, N), np.float16)
        assert lib.hqq_b200_linear_fwd_route(i64(M), i64(N), i64(K), gs, nbits, 1, R.F16) == 2
        nb = lib.hqq_b200_linear_fwd_workspace_bytes(M, N, K, gs, nbits, 1, R.F16)
        ws = R.aligned((max(nb, 1),), np.uint8)
        ws[...] = 0xCD  # scratch arrives dirty
        for rep in range(2):
            y[...] = 0
            rc = lib.hqq_b200_linear_fwd(R.P(xd), R.P(L["Wq"]), R.P(L["scale"]), R.P(L["zero"]), R.P(L["bias"]), R.P(y), i64(M), i64(N), i64(K), gs, nbits,
                                         1, R.F16, R.P(ws) if nb else None, ctypes.c_size_t(nb), None)
            assert rc == 0, lib.hqq_b200_last_error()
            res[f"gemm{ci}" + ("_again" if rep else "")] = y.copy()
        res[f"gemm{ci}_ws"] = np.array([nb])
        res[f"gemm{ci}_ref"] = O.linear_forward(x.astype(np.float32), L["Wq_host"], L["meta"], None if not wb else L["bias_host"].astype(np.float32),
                                                "float16")
    for ci, (nbits, gs, N, K, M, wb) in enumerate(DENSE_CASES):
        rng = np.random.default_rng(900 + ci)
        L = R.make_layer(rng, N, K, nbits, gs, wb)
        x = rng.standard_normal((M, K)).astype(np.float16)
        xd, y = R.dev(x), R.aligned((M, N), np.float16)
        assert lib.hqq_b200_linear_fwd_route(i64(M), i64(N), i64(K), gs, nbits, 1, R.F16) == 3, (nbits, gs, N, K, M)
        nb = lib.hqq_b200_linear_fwd_workspace_bytes(M, N, K, gs, nbits, 1, R.F16)
        assert nb >= N * K * 2
        ws = R.aligned((nb,), np.uint8)
        ws[...] = 0xCD
        rc = lib.hqq_b200_linear_fwd(R.P(xd), R.P(L["Wq"]), R.P(L["scale"]), R.P(L["zero"]), R.P(L["bias"]), R.P(y), i64(M), i64(N), i64(K), gs, nbits,
                                     1, R.F16, R.P(ws), ctypes.c_size_t(nb), None)
        assert rc == 0, lib.hqq_b200_last_error()
        res[f"dense{ci}"] = y.copy()
        res[f"dense{ci}_ref"] = O.linear_forward(x.astype(np.float32), L["Wq_host"], L["meta"], None if not wb else L["bias_host"].astype(np.float32),
                                                 "float16")
    np.savez(out_path, **res)


if __name__ == "__main__":
    main(sys.argv[1])
