"""CPU: the C-ABI library loads, exports every symbol include/hqq_b200.h declares, and validates its
arguments before touching the GPU (no compute happens in this file)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from hqq_b200 import build, _lib
    build.build()
    return _lib.load()


def header_symbols():
    src = open(os.path.join(ROOT, "include", "hqq_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(hqq_b200_\w+)\s*\(", src)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    from hqq_b200 import _lib
    syms = header_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/hqq_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes prototype"
    assert sorted(_lib.SIGNATURES) == syms


def test_abi_version(lib):
    assert lib.hqq_b200_abi_version() == 2


def test_argument_validation_uses_reference_wording(lib):
    from hqq_b200 import _lib
    # unsupported bit width
    rc = lib.hqq_b200_pack(5, None, 0, None, 8, 8, None)
    assert rc == _lib.HQQ_E_INVALID and "not supported" in _lib.last_error()
    # ragged slab split (the reference fails on W_q[:step] | W_q[step:])
    rc = lib.hqq_b200_pack(4, 1, _lib.HQQ_U8, 1, 7, 8, None)
    assert rc == _lib.HQQ_E_INVALID
    # group size must divide the tensor (quantize.py:92-100 wording)
    assert lib.hqq_b200_quantize_workspace_bytes(10, 10, 64, 4, 1, 20) == 0
    rc = lib.hqq_b200_quantize(None, 0, 10, 10, 64, 4, 1, 0, 1, 0.7, 10.0, 20, None, None, None, None, None, None, 0, None)
    assert rc == _lib.HQQ_E_INVALID and "group_size should be divisble" in _lib.last_error()
    rc = lib.hqq_b200_dequantize(1, 1, 1, 1, 64, 64, 64, 4, 2, _lib.HQQ_F16, None)
    assert rc == _lib.HQQ_E_INVALID and "axis should be either 0 or 1" in _lib.last_error()
    # workspace size is a pure function of the shape
    assert lib.hqq_b200_quantize_workspace_bytes(4096, 4096, 64, 4, 1, 20) > 4096 * 4096 // 64 * 4 * 21


def test_forward_routing_table(lib):
    from hqq_b200._lib import HQQ_BF16, HQQ_F16, HQQ_F32
    r = lib.hqq_b200_linear_fwd_route
    assert r(1, 4096, 4096, 64, 4, 1, HQQ_F16) == 1      # decode: weight-streaming kernel
    assert r(16, 14336, 4096, 64, 4, 1, HQQ_BF16) == 1   # up to 16 tokens the weight-streaming kernel wins on every matrix
    assert r(32, 4096, 4096, 64, 4, 1, HQQ_BF16) == 1    # 17..32 tokens: still on matrices up to 4096 x 4096 ...
    assert r(32, 14336, 4096, 64, 4, 1, HQQ_BF16) == 2   # ... larger ones go to the wgmma kernel (boundary rule, linear.cu)
    assert r(17, 4096, 14336, 64, 4, 1, HQQ_F16) == 2
    assert r(32, 3584, 8192, 64, 4, 1, HQQ_F16) == 2 and r(32, 1280, 8192, 64, 4, 1, HQQ_F16) == 1   # the boundary: 2^24 weights
    assert r(32, 14336, 4096, 64, 4, 1, HQQ_F32) == 0
    assert r(1, 4096, 4096, 64, 4, 0, HQQ_F16) == 3      # axis 0: dequantize kernel + dense wgmma GEMM
    assert r(1, 4096, 4096, 64, 4, 1, HQQ_F32) == 0      # float32 compute: no tensor-core route
    assert r(1, 4096, 4096, 64, 3, 1, HQQ_F16) == 3      # 3-bit (ten fields per int32, slabs cut rows): route 3
    assert r(1, 4096, 4000, 64, 4, 1, HQQ_F16) == 3      # the fused kernels need K % 256 == 0; the dense GEMM's TMA zero-fills ragged K
    assert r(1, 4096, 4096, 128, 2, 1, HQQ_BF16) == 1
    assert r(1, 4096, 4096, 32, 4, 1, HQQ_F16) == 3      # group sizes other than 64/128
    assert r(4096, 4096, 4096, 64, 4, 1, HQQ_F16) == 2   # fused wgmma GEMM
    wsb = lib.hqq_b200_linear_fwd_workspace_bytes
    assert wsb(1, 4096, 4096, 64, 4, 1, HQQ_F16) == 0 and wsb(4096, 4096, 4096, 64, 4, 1, HQQ_F16) == 0
    assert wsb(128, 4096, 4096, 64, 4, 1, HQQ_F16) % (32 * 256 * 128 * 4) == 0 and wsb(128, 4096, 4096, 64, 4, 1, HQQ_F16) > 0  # few tiles: split-K partials
    assert wsb(64, 4096, 4096, 64, 3, 1, HQQ_F16) == 4096 * 4096 * 2 and wsb(64, 4096, 4096, 64, 4, 0, HQQ_BF16) == 4096 * 4096 * 2
    assert r(64, 4096, 4096, 64, 4, 1, HQQ_F16) != 1     # beyond the small-M kernel


def test_missing_library_fails_loudly(tmp_path):
    from hqq_b200 import _lib
    with pytest.raises(RuntimeError, match="no CPU or PyTorch fallback"):
        _lib.load(str(tmp_path / "nope.so"))


def test_decode_desc_ctypes_mirror_matches_the_c_struct(tmp_path):
    """`hqq_b200_decode_desc` (include/hqq_b200.h) against its ctypes mirror (hqq_b200/_lib.py): same size, same field names and
    offsets -- compiled with the system C compiler, so a drifting header or mirror fails here and not as a wild pointer on the GPU."""
    import ctypes
    import shutil
    import subprocess
    from hqq_b200._lib import DecodeDesc
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = [f[0] for f in DecodeDesc._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "hqq_b200.h"\nint main(void) {\n'
                   '  printf("sizeof %zu\\n", sizeof(hqq_b200_decode_desc));\n'
                   + "".join(f'  printf("{n} %zu\\n", offsetof(hqq_b200_decode_desc, {n}));\n' for n in names) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run([cc, "-x", "c", "-std=c11", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["sizeof"]) == ctypes.sizeof(DecodeDesc)
    for n in names:
        assert int(out[n]) == getattr(DecodeDesc, n).offset, n
