"""TEST INFRASTRUCTURE ONLY: `hqq_b200_reload_env()` on the emulated library -- the HQQ_B200_* knobs are cached per process and
parsed again only after a reload.  Observable without a GPU or a launch: HQQ_B200_GEMM_CTAS sets the number of persistent CTAs
the route-2 schedule is built for, and with it the split-K workspace `hqq_b200_linear_fwd_workspace_bytes` asks for.  The
emulator reports 4 SMs, so M = 64, N = 128, K = 1024 (4-bit, gs 64: one output tile) splits K four ways by default and not at
all with HQQ_B200_GEMM_CTAS=1.  Prints one JSON line."""
import ctypes
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_emu  # noqa: E402
from run_small import F16  # noqa: E402


def main():
    for k in [k for k in os.environ if k.startswith("HQQ_B200_")]:
        del os.environ[k]
    lib = ctypes.CDLL(build_emu.build())
    lib.hqq_b200_linear_fwd_workspace_bytes.restype = ctypes.c_size_t
    i64 = ctypes.c_int64
    M, N, K, gs, nbits = 64, 128, 1024, 64, 4
    assert lib.hqq_b200_linear_fwd_route(i64(M), i64(N), i64(K), gs, nbits, 1, F16) == 2

    def ws():
        return int(lib.hqq_b200_linear_fwd_workspace_bytes(i64(M), i64(N), i64(K), gs, nbits, 1, F16))

    out = {"default_ws": ws()}
    os.environ["HQQ_B200_GEMM_CTAS"] = "1"
    out["cached_ws"] = ws()                                      # knob changed, no reload: still the cached CTA count
    lib.hqq_b200_reload_env()
    out["reloaded_ws"] = ws()                                    # one CTA: no k-slices, no workspace
    del os.environ["HQQ_B200_GEMM_CTAS"]
    lib.hqq_b200_reload_env()
    out["restored_ws"] = ws()
    print("RELOAD " + json.dumps(out))


if __name__ == "__main__":
    main()
