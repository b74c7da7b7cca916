"""CPU: the kernels of hqq_b200/csrc EXECUTED on the CPU by the cooperative-fiber emulator in tests/emu (every CUDA thread a fiber,
warp collectives and __syncthreads as rendezvous; mbarrier / TMA / wgmma / cp.async / mma.sync as functional models)
and compared with the oracle and the reference's fixtures.

Why: kernels are written in a container without a GPU.  This executes the very same source text (two syntactic rewrites, see
tests/emu/build_emu.py) so that indexing, control flow, barrier protocols and the collectives' use are checked before a GPU run.
It says nothing about performance, async proxies or memory ordering.  The emulator is test infrastructure: the product library
has no CPU path, and this one is loaded here through ctypes only."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
F32, F16, BF16, U8, I32 = 0, 1, 2, 3, 4


@pytest.fixture(scope="module")
def emu():
    import build_emu
    try:
        lib = ctypes.CDLL(build_emu.build())
    except RuntimeError as e:  # no g++ / CUDA headers: nothing to emulate with
        pytest.skip(f"emulator build unavailable: {str(e)[:200]}")
    lib.hqq_b200_quantize_workspace_bytes.restype = ctypes.c_size_t
    lib.hqq_b200_quantize_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.hqq_b200_last_error.restype = ctypes.c_char_p
    return lib


def P(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def aligned(shape, dtype, align=256):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.zeros(n + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + n].view(dtype).reshape(shape)


def to_bf16_bits(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


def quantize(lib, W, src, nbits, gs, variant, lp=0.7, iters=20, axis=1, optimize=1):
    N, K = W.shape
    if src == F16:
        Wd = aligned(W.shape, np.float16); Wd[...] = W.astype(np.float16)
    elif src == BF16:
        Wd = aligned(W.shape, np.uint16); Wd[...] = to_bf16_bits(W)
    else:
        Wd = aligned(W.shape, np.float32); Wd[...] = W
    G = N * K // gs
    fields = 10 if nbits == 3 else 8 // nbits
    R, C = (G, gs) if axis == 1 else (gs, G)  # the grouped view [R, C]; packing runs along R
    prow = -(-R // 10) if nbits == 3 else R // fields
    Wq = aligned((prow, C), np.int32 if nbits == 3 else np.uint8)
    s, z = aligned((G,), np.float32), aligned((G,), np.float32)
    info, err = aligned((4,), np.int32), aligned((iters,), np.float32)
    nb = lib.hqq_b200_quantize_workspace_bytes(N, K, gs, nbits, axis, iters)
    assert nb > 0
    ws = aligned((nb,), np.uint8)
    # variant 0: the plain 20-iteration loop (solver_generic_kernel, HQQ_B200_PLAIN_SOLVER=1); 1: the register-resident default
    if variant == 0:
        os.environ["HQQ_B200_PLAIN_SOLVER"] = "1"
    try:
        rc = lib.hqq_b200_quantize(P(Wd), src, ctypes.c_int64(N), ctypes.c_int64(K), gs, nbits, axis, int(nbits == 4), int(optimize), ctypes.c_float(lp),
                                   ctypes.c_float(10.0), iters, P(Wq), P(s), P(z), P(info), P(err), P(ws), ctypes.c_size_t(nb), None)
    finally:
        os.environ.pop("HQQ_B200_PLAIN_SOLVER", None)
    assert rc == 0, lib.hqq_b200_last_error()
    return Wq.copy(), s.copy(), z.copy(), info.copy(), err.copy(), Wd


def test_emulated_pack_unpack_dequantize_match_the_oracle(emu, oracle):
    rng = np.random.default_rng(0)
    for nbits in (8, 4, 3, 2, 1):
        rows, cols = 40, 24
        q = rng.integers(0, 2 ** nbits, size=(rows, cols)).astype(np.uint8)
        packing = oracle.BIT_TO_PACKING[nbits]
        ref = oracle.PACK[packing](q)
        qd = aligned(q.shape, np.uint8); qd[...] = q
        out = aligned(ref.shape, ref.dtype)
        assert emu.hqq_b200_pack(nbits, P(qd), U8, P(out), ctypes.c_int64(rows), ctypes.c_int64(cols), None) == 0, emu.hqq_b200_last_error()
        assert np.array_equal(out, ref), nbits
        back = aligned((ref.shape[0] * (10 if nbits == 3 else 8 // nbits), cols), np.uint8)
        assert emu.hqq_b200_unpack(nbits, P(out), P(back), U8, ctypes.c_int64(ref.shape[0]), ctypes.c_int64(cols), None) == 0
        assert np.array_equal(back[:rows], q), nbits


@pytest.mark.parametrize("nbits,gs,shape,std", [(4, 64, (32, 256), 0.02), (2, 32, (16, 128), 0.5), (3, 64, (25, 128), 0.02)])
def test_emulated_default_solver_matches_the_oracle(emu, oracle, nbits, gs, shape, std):
    """Pins the emulator itself: the DEFAULT solver kernel, which the GPU suite validates against the oracle, must agree with
    the oracle here to the same tolerances (tests/test_quantize_gpu.py)."""
    rng = np.random.default_rng(nbits)
    W = (rng.standard_normal(shape) * std).astype(np.float32)
    Wq, s, z, info, err, _ = quantize(emu, W, F32, nbits, gs, 0)
    ref_Wq, ref_meta = oracle.quantize(W, nbits=nbits, group_size=gs, axis=1, optimize=True, round_zero=(nbits == 4))[:2]
    ref_q = oracle.UNPACK[ref_meta["packing"]](ref_Wq)[: W.size // gs]
    got_q = oracle.UNPACK[ref_meta["packing"]](Wq)[: W.size // gs]
    assert np.array_equal(s, ref_meta["scale"].ravel())
    # float64 zero-point sums in the kernel and in the oracle: identical levels, zero-points equal to the last bit (the residual
    # arithmetic differences -- (W_q - z) * (1/s) for the division, ex2/lg2 for pow -- only touch the error sums and W_e != 0)
    assert np.array_equal(got_q, ref_q)
    assert np.allclose(z, ref_meta["zero"].ravel(), rtol=0, atol=1e-6 * max(1.0, float(np.abs(z).max())))


@pytest.mark.parametrize("variant", [0, 1])
def test_emulated_solver_reproduces_every_level_of_the_reference_fixtures(emu, oracle, golden, variant):
    """The solver kernels' own source on the emulator against the fixtures the REAL reference produced (tests/golden): identical
    iteration counts and identical levels on all 14 configurations (both axes, five widths, three group sizes), for the default
    and the fast solver.  (Before the zero-point means were accumulated in float64 the kernels differed in 2 of 393 216 levels.)"""
    q = golden.quant
    for nbits in (8, 4, 3, 2, 1):
        for axis in (0, 1):
            for gs in ((64,) if nbits != 4 else (64, 32, 128)):
                if variant == 1 and (nbits, axis, gs) not in ((4, 1, 64), (4, 0, 64), (3, 1, 64), (8, 0, 64), (4, 1, 128)):
                    continue  # the fast solver is bit-identical to the default one (separate test): a subset keeps the suite short
                key = f"b{nbits}_a{axis}_g{gs}"
                Wq, s, z, info, err, _ = quantize(emu, q["W"], F32, nbits, gs, variant, axis=axis)
                pk = oracle.BIT_TO_PACKING[nbits]
                rows = q["W"].size // gs if axis == 1 else gs
                assert int(info[0]) == int(q[key + "/iters"]), key
                assert np.array_equal(oracle.UNPACK[pk](Wq)[:rows], oracle.UNPACK[pk](q[key + "/W_q"])[:rows]), key
                assert np.array_equal(s, q[key + "/scale"].ravel()), key
                zr = q[key + "/zero"].ravel()
                assert np.max(np.abs(z - zr) / np.maximum(np.abs(zr), 1.0)) <= 1e-6, key


CASES = [(4, 64, (32, 256), 0.02, F16), (4, 64, (30, 128), 1.0, F16),   # std 1.0: |W - W_r| above the threshold, the fallback runs
         (2, 64, (16, 256), 0.02, BF16), (2, 32, (16, 128), 2.0, F32), (8, 128, (16, 256), 0.05, F16), (1, 16, (16, 64), 0.02, F32),
         (3, 64, (25, 128), 0.02, F16), (4, 8, (12, 64), 0.5, F32), (4, 256, (8, 512), 0.02, F16), (4, 64, (19, 128), 0.02, F16)]


@pytest.mark.parametrize("nbits,gs,shape,std,src", CASES)
@pytest.mark.parametrize("lp", [0.7, 1.0])
def test_emulated_register_solver_equals_the_plain_loop(emu, nbits, gs, shape, std, src, lp):
    rng = np.random.default_rng(nbits * 100 + gs)
    W = (rng.standard_normal(shape) * std).astype(np.float32)
    a = quantize(emu, W, src, nbits, gs, 0, lp)
    b = quantize(emu, W, src, nbits, gs, 1, lp)
    # levels, scale, zero-points and the iteration count are bit-identical; the per-iteration error means come from a different
    # (equally fixed) float32 summation order in the plain one-warp-per-group loop, hence the last-bit tolerance on them only
    assert np.allclose(a[4], b[4], rtol=2e-6, atol=0), "errors"
    assert np.array_equal(a[1], b[1]), "scale"
    if int(a[3][0]) == int(b[3][0]):
        for x, y, what in zip(a[:4], b[:4], ("W_q", "scale", "zero", "info")):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), what
    else:
        # two consecutive error means tie to the last float32 bit and the two summation orders break the tie differently: the early
        # stop fires one iteration apart (the reference's own torch.mean has a third order) -- zero-points then differ by one update
        assert abs(int(a[3][0]) - int(b[3][0])) == 1
        k = min(int(a[3][0]), int(b[3][0]))
        assert abs(float(a[4][k - 1]) - float(a[4][k - 2])) <= 4e-7 * float(a[4][k - 1])
    assert 1 <= a[3][0] <= 20


@pytest.mark.parametrize("nbits,gs,shape,std,src", [(4, 64, (64, 48), 0.02, F16), (4, 64, (64, 33), 1.0, F32), (2, 32, (32, 100), 0.02, BF16),
                                                    (8, 16, (16, 70), 0.05, F16), (3, 8, (8, 90), 0.5, F32), (1, 64, (128, 40), 0.02, F16)])
@pytest.mark.parametrize("lp", [0.7, 1.0])
def test_emulated_register_solver_axis0_equals_the_plain_loop(emu, nbits, gs, shape, std, src, lp):
    rng = np.random.default_rng(nbits * 10 + gs)
    W = (rng.standard_normal(shape) * std).astype(np.float32)
    a = quantize(emu, W, src, nbits, gs, 0, lp, axis=0)
    b = quantize(emu, W, src, nbits, gs, 1, lp, axis=0)
    # levels, scale, zero-points and the iteration count are bit-identical; the per-iteration error means come from a different
    # (equally fixed) float32 summation order in the plain one-warp-per-group loop, hence the last-bit tolerance on them only
    assert np.allclose(a[4], b[4], rtol=2e-6, atol=0), "errors"
    assert np.array_equal(a[1], b[1]), "scale"
    if int(a[3][0]) == int(b[3][0]):
        for x, y, what in zip(a[:4], b[:4], ("W_q", "scale", "zero", "info")):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), what
    else:
        # two consecutive error means tie to the last float32 bit and the two summation orders break the tie differently: the early
        # stop fires one iteration apart (the reference's own torch.mean has a third order) -- zero-points then differ by one update
        assert abs(int(a[3][0]) - int(b[3][0])) == 1
        k = min(int(a[3][0]), int(b[3][0]))
        assert abs(float(a[4][k - 1]) - float(a[4][k - 2])) <= 4e-7 * float(a[4][k - 1])


# ---------------------------------------------------------------------------------------------------------------------------
# The headline kernels: csrc/linear_small.cu (generic small-M kernel and the one-token kernel) on the emulator.  mma.sync,
# prmt, lop3 and cp.async are emulated (tests/emu/include/cuda_runtime.h); the kernel source is the product's, with its inline
# PTX switched to those stand-ins by -DHQQ_EMU (the GPU build's SASS is byte-identical with and without the #ifdefs).
# ---------------------------------------------------------------------------------------------------------------------------
import subprocess  # noqa: E402

RUNNER = os.path.join(HERE, "emu", "run_small.py")
_RUNS = {}


def run_small(tmp_path_factory):
    key = "default"
    if key not in _RUNS:
        out = str(tmp_path_factory.mktemp("emu_small") / f"{key}.npz")
        env = {k: v for k, v in os.environ.items() if not k.startswith("HQQ_B200_")}
        r = subprocess.run([sys.executable, RUNNER, out], env=env, capture_output=True, text=True, timeout=600)
        if r.returncode != 0:
            if "emulator build unavailable" in r.stderr or "g++" in r.stderr and "not found" in r.stderr:
                pytest.skip("emulator build unavailable")
            raise AssertionError(r.stderr[-3000:])
        _RUNS[key] = dict(np.load(out))
    return _RUNS[key]


def rel(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def test_emulated_small_m_and_one_token_forward_match_the_oracle(emu, tmp_path_factory):
    d = run_small(tmp_path_factory)
    refs = [k for k in d if k.endswith("_ref")]
    assert len(refs) >= 20
    for k in refs:
        assert rel(d[k[:-4]], d[k]) <= 2e-3, k  # fp16 tolerance of tests/test_linear_gpu.py (measured there and here: ~3e-4)


def test_emulated_one_token_prologues_and_paired_epilogue(emu, oracle, tmp_path_factory):
    """x_op 1 (residual add + RMSNorm), x_op 2 (SiLU * mul) and the paired SiLU*mul epilogue against numpy restatements of the
    documented roundings (include/hqq_b200.h: every intermediate is rounded to the compute dtype)."""
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import run_small as R
    d = run_small(tmp_path_factory)
    f16 = lambda v: np.asarray(v, dtype=np.float32).astype(np.float16)  # noqa: E731
    silu = lambda v: f16(v.astype(np.float32) / (1.0 + np.exp(-v.astype(np.float32))))  # noqa: E731
    for ci, (nbits, N, K) in enumerate(R.DECODE):
        rng = np.random.default_rng(200 + ci)
        A, B = R.make_layer(rng, N, K, nbits, 64), R.make_layer(rng, N, K, nbits, 64)
        x = rng.standard_normal((1, K)).astype(np.float16)
        x2 = (rng.standard_normal((1, K)) * 0.5).astype(np.float16)
        w = rng.random(K).astype(np.float16)
        fwd = lambda act, L: oracle.linear_forward(act.astype(np.float32), L["Wq_host"], L["meta"], None, "float16")  # noqa: E731
        # x_op 1
        t = f16(x.astype(np.float32) + x2.astype(np.float32))
        inv = 1.0 / np.sqrt(np.mean(t.astype(np.float32) ** 2) + 1e-5)
        xn = f16(f16(t.astype(np.float32) * np.float32(inv)).astype(np.float32) * w.astype(np.float32))
        assert np.array_equal(d[f"dec{ci}_x1_h"], t)
        assert rel(d[f"dec{ci}_x1_a"], fwd(xn, A)) <= 3e-3 and rel(d[f"dec{ci}_x1_b"], fwd(xn, B)) <= 3e-3
        # x_op 2
        xm = f16(silu(x).astype(np.float32) * x2.astype(np.float32))
        assert rel(d[f"dec{ci}_x2_a"], fwd(xm, A)) <= 3e-3
        # paired epilogue on the plain activation: silu(W0 x) * (W1 x), both products rounded first
        g, u = d[f"dec{ci}_x0_a"], d[f"dec{ci}_x0_b"]
        assert np.array_equal(d[f"dec{ci}_x0pair_a"], f16(silu(g).astype(np.float32) * u.astype(np.float32)))
        g1, u1 = d[f"dec{ci}_x1_a"], d[f"dec{ci}_x1_b"]
        assert np.array_equal(d[f"dec{ci}_x1pair_a"], f16(silu(g1).astype(np.float32) * u1.astype(np.float32)))
        assert np.array_equal(d[f"dec{ci}_x1pair_h"], t)


# ---------------------------------------------------------------------------------------------------------------------------
# csrc/linear_gemm.cu on the emulator's functional model of mbarrier / TMA (SWIZZLE_128B) / wgmma descriptors / wgmma.mma_async
# register fragments / wait_group: addresses, swizzles, barrier phases and who-waits-for-whom are executed; timing, async proxies and memory
# ordering are not.  A barrier protocol that cannot make progress is reported as a deadlock by the scheduler.
# ---------------------------------------------------------------------------------------------------------------------------
GEMM_RUNNER = os.path.join(HERE, "emu", "run_gemm.py")
_GEMM = {}


def run_gemm_emu(tmp_path_factory, knob=None, async_seed=None):
    key = ("default" if knob is None else "=".join(knob)) + (f"@{async_seed}" if async_seed is not None else "")
    if key not in _GEMM:
        out = str(tmp_path_factory.mktemp("emu_gemm") / "out.npz")
        env = {k: v for k, v in os.environ.items() if not k.startswith("HQQ_B200_") and not k.startswith("EMU_")}
        if knob:
            env[knob[0]] = knob[1]
        if async_seed is not None:  # adversarial timing: asynchronous operations land 0..8 scheduler passes late, threads in random order
            env["EMU_ASYNC"], env["EMU_SEED"] = "8", str(async_seed)
        r = subprocess.run([sys.executable, GEMM_RUNNER, out], env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        _GEMM[key] = dict(np.load(out))
    return _GEMM[key]


def test_emulated_tcgen05_gemm_matches_the_oracle(emu, tmp_path_factory):
    d = run_gemm_emu(tmp_path_factory)
    refs = [k for k in d if k.endswith("_ref") and k.startswith("gemm")]
    assert len(refs) == 12
    dense = [k for k in d if k.endswith("_ref") and k.startswith("dense")]
    assert len(dense) == 5
    for k in dense:  # route 3: W_r from the dequantize kernel (the reference's two roundings), dense wgmma GEMM, fp32 accumulation
        assert rel(d[k[:-4]], d[k]) <= 1e-4, k
    for k in refs:
        # the A operand is dequantised with the reference's two roundings and accumulated in fp32: far inside the fp16 tolerance
        assert rel(d[k[:-4]], d[k]) <= 1e-4, k
        assert np.array_equal(d[k[:-4]], d[k[:-4] + "_again"]), k  # also on a dirty split-K workspace: deterministic
    assert sum(int(d[k[:-4] + "_ws"][0]) > 0 for k in refs) >= 1  # few tiles x long K: k-slices + second-pass reduction


@pytest.mark.parametrize("knob", [("HQQ_B200_GEMM_CTAS", "1"), ("HQQ_B200_GEMM_CTAS", "3"), ("HQQ_B200_GEMM_CTAS", "5"), ("HQQ_B200_GEMM_CTAS", "24")])
def test_emulated_persistent_gemm_schedules_are_bit_identical(emu, tmp_path_factory, knob):
    """The persistent kernel with its grid capped to 1 / 3 / 5 CTAs: every CTA then walks several tiles (accumulators reused,
    epilogue of tile i under the main loop of tile i + 1, rings running across tile boundaries, the half-tile round of the
    schedule) and issues the same MMAs in the same k order per output element as the one-tile-per-CTA run: identical outputs,
    and no barrier protocol that stalls."""
    ref, got = run_gemm_emu(tmp_path_factory), run_gemm_emu(tmp_path_factory, knob)
    for k in ref:
        if k.endswith("_ws"):
            continue
        base = k[:-6] if k.endswith("_again") else (k[:-4] if k.endswith("_ref") else k)
        split = (base + "_ws") in ref and (int(ref[base + "_ws"][0]) > 0 or int(got[base + "_ws"][0]) > 0)
        if split and not k.endswith("_ref"):  # the number of k-slices follows the CTA count: fp32 summation order differs
            assert rel(got[k], ref[k]) <= 1e-4, k
        else:
            assert np.array_equal(ref[k].view(np.uint8), got[k].view(np.uint8)), k


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_emulated_persistent_gemm_under_adversarial_timing(emu, tmp_path_factory, seed):
    """EMU_ASYNC: TMA copies, tensor-core operations and their commits land a random number of scheduler passes late and threads
    resume in random order; the capped grid keeps several tiles per CTA in flight.  Same bits as the in-order run."""
    ref = run_gemm_emu(tmp_path_factory, ("HQQ_B200_GEMM_CTAS", "2"))
    got = run_gemm_emu(tmp_path_factory, ("HQQ_B200_GEMM_CTAS", "2"), async_seed=seed)
    for k in ref:
        assert np.array_equal(ref[k].view(np.uint8), got[k].view(np.uint8)), k


@pytest.mark.parametrize("tp", [2, 8])
def test_emulated_tensor_parallel_exchange(emu, tmp_path, tp):
    """The fused all-reduce (tagged words over peer memory, csrc/linear_small.cu) with `tp` ranks as `tp` buffer sets in one process:
    every rank's buffer receives every rank's partial in slot [parity][rank][n] with the exchange's tag, the consumer's fp32
    reduction in rank order + residual add reproduce numpy bit for bit, and the next linear sees the right activation -- over
    three steps x two blocks, so tags and parities roll.  tp = 8 has not run on GPUs yet; this is its data path."""
    r = subprocess.run([sys.executable, os.path.join(HERE, "emu", "run_tp.py"), str(tp), str(tmp_path / "tp.npz")], capture_output=True, text=True,
                       timeout=900, env={k: v for k, v in os.environ.items() if not k.startswith("HQQ_B200_")})
    assert r.returncode == 0, r.stderr[-3000:]
    d = np.load(str(tmp_path / "tp.npz"))
    assert len(d.files) == 3 * 2 * tp


def test_emulated_forward_random_shapes(emu, oracle):
    """Seeded sweep over what the router accepts (4/2/1/8-bit, gs 64/128, K a multiple of 256, M = 1..300, ragged N, bias or not):
    whichever kernel hqq_b200_linear_fwd picks -- one-token, generic small-M or wgmma GEMM -- must agree with the oracle.  600
    further configurations from other seeds were run while developing this; none exceeded 5.4e-4."""
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import run_small as R
    rng = np.random.default_rng(7)
    i64 = ctypes.c_int64
    routes = set()
    for _ in range(40):
        nbits = int(rng.choice([8, 4, 2, 1])); gs = int(rng.choice([64, 128])); F = 8 // nbits
        K = 256 * int(rng.integers(1, 7))
        M = int(rng.integers(1, 33)) if rng.random() < 0.5 else int(rng.integers(33, 300))
        N = F * int(rng.integers(1, 48))
        wb = bool(rng.random() < 0.5)
        L = R.make_layer(rng, N, K, nbits, gs, wb)
        x = rng.standard_normal((M, K)).astype(np.float16)
        xd, y = R.dev(x), R.aligned((M, N), np.float16)
        route = emu.hqq_b200_linear_fwd_route(i64(M), i64(N), i64(K), gs, nbits, 1, F16)
        assert route in (1, 2)
        routes.add(route)
        emu.hqq_b200_linear_fwd_workspace_bytes.restype = ctypes.c_size_t
        nws = int(emu.hqq_b200_linear_fwd_workspace_bytes(i64(M), i64(N), i64(K), gs, nbits, 1, F16))  # > 0: few tiles, split-K partials
        ws = R.aligned((max(nws, 1),), np.uint8)
        ws[:] = 0xA5  # contents on entry are irrelevant
        rc = emu.hqq_b200_linear_fwd(R.P(xd), R.P(L["Wq"]), R.P(L["scale"]), R.P(L["zero"]), R.P(L["bias"]), R.P(y), i64(M), i64(N), i64(K), gs, nbits, 1,
                                     F16, R.P(ws) if nws else None, ctypes.c_size_t(nws), None)
        assert rc == 0, emu.hqq_b200_last_error()
        ref = oracle.linear_forward(x.astype(np.float32), L["Wq_host"], L["meta"], None if not wb else L["bias_host"].astype(np.float32), "float16")
        assert rel(y, ref) <= 2e-3, (nbits, gs, N, K, M, wb, route)
    assert routes == {1, 2}


def test_emulated_reload_env_switches_cached_knobs_in_one_process(emu):
    """`hqq_b200_reload_env()`: a changed HQQ_B200_* switch is ignored until the reload and honoured after it."""
    import json
    r = subprocess.run([sys.executable, os.path.join(HERE, "emu", "run_reload.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RELOAD ")][-1][7:])
    assert out["default_rc"] == 0
    assert out["cached_rc"] == 0 and out["cached_same"]          # no reload: the cached choice stands
    assert out["reloaded_rc"] == -2                              # HQQ_E_UNSUPPORTED once HQQ_B200_DECODE1=0 is seen
    assert out["restored_rc"] == 0 and out["restored_same"]


@pytest.mark.parametrize("variant,cases", [(0, [(4, 0), (4, 1), (2, 0), (2, 1), (1, 0), (1, 1)]), (1, [(4, 1), (2, 0)])])
def test_emulated_solver_on_the_heavy_tailed_reference_fixture(emu, oracle, golden, variant, cases):
    """Weights whose quantisation error exceeds the shrinkage threshold (the full formula with ex2/lg2 runs, the fast solver takes
    its fallback): the kernels' source still reproduces the reference's iteration counts and every level."""
    h = golden.heavy
    for nbits, axis in cases:
        key = f"b{nbits}_a{axis}_g64"
        Wq, s, z, info, err, _ = quantize(emu, h["W"], F32, nbits, 64, variant, axis=axis)
        pk = oracle.BIT_TO_PACKING[nbits]
        rows = h["W"].size // 64 if axis == 1 else 64
        assert int(info[0]) == int(h[key + "/iters"]), key
        assert np.array_equal(oracle.UNPACK[pk](Wq)[:rows], oracle.UNPACK[pk](h[key + "/W_q"])[:rows]), key
        zr = h[key + "/zero"].ravel()
        assert np.max(np.abs(z - zr) / np.maximum(np.abs(zr), 1.0)) <= 2e-6, key


@pytest.mark.parametrize("nbits", (4, 2, 8))
def test_emulated_quantizer_on_the_degenerate_reference_fixture(emu, oracle, golden, nbits):
    """Groups on the guards of the init (constant, boundary of the 1e-4 test, clamped inverse scale, huge range, zeros): the
    kernels' init + rounding path is bit-exact against the reference; with the solver on, the scale stays bit-exact, at most one
    level of the 768 moves and the zero-points agree to 2e-6 -- the same statement as for the oracles."""
    d = golden.degenerate
    pk = oracle.BIT_TO_PACKING[nbits]
    Wq, s, z, info, err, _ = quantize(emu, d["W"], F32, nbits, 64, 0, optimize=0)
    assert np.array_equal(Wq, d[f"b{nbits}_opt0/W_q"])
    assert np.array_equal(s, d[f"b{nbits}_opt0/scale"].ravel()) and np.array_equal(z, d[f"b{nbits}_opt0/zero"].ravel())
    for variant in (0, 1):
        Wq, s, z, info, err, _ = quantize(emu, d["W"], F32, nbits, 64, variant)
        a, b = oracle.UNPACK[pk](Wq).astype(int), oracle.UNPACK[pk](d[f"b{nbits}_opt1/W_q"]).astype(int)
        assert np.abs(a - b).max() <= 1 and (a != b).sum() <= 1, variant
        assert np.array_equal(s, d[f"b{nbits}_opt1/scale"].ravel())
        zr = d[f"b{nbits}_opt1/zero"].ravel()
        assert np.all(np.isfinite(z)) and np.max(np.abs(z - zr) / np.maximum(np.abs(zr), 1.0)) <= 2e-6, variant


def test_emulated_solver_equals_the_c_oracle_on_random_layers(emu, oracle):
    """Random layers (both axes, four widths, three group sizes): the solver kernels' source, run on the emulator, against the
    C oracle (which reproduces the reference's fixtures level for level, tests/test_oracle_c.py).  Weight-like data (the shrinkage
    is exactly zero): identical iteration counts and levels.  Heavy-tailed data (W_e != 0, where the kernel's ex2/lg2 and
    reciprocal differ from powf and the division at the 1e-7 level): the GPU tests' tolerance."""
    try:
        from oracle import hqq_oracle_c as C
        C.lib()
    except (RuntimeError, OSError) as e:
        pytest.skip(f"C oracle cannot be built here: {e}")
    rng = np.random.default_rng(2024)
    exact = 0
    for case in range(14):
        nbits = (4, 2, 8, 1, 3, 4, 4)[case % 7]
        gs = (64, 32, 128)[case % 3]
        axis = case % 2
        heavy = case >= 11
        N, K = int(rng.integers(2, 6)) * 16, int(rng.integers(1, 4)) * 128
        W = (rng.standard_normal((N, K)) * (1.5 if heavy else 0.02) + (0.01 if case % 4 == 0 else 0.0)).astype(np.float32)
        rows = N * K // gs if axis == 1 else gs
        if nbits != 3 and rows % (8 // nbits):
            continue
        Wq, s, z, info, err, _ = quantize(emu, W, F32, nbits, gs, case % 2, axis=axis)
        Wq_c, meta_c, tr_c = C.quantize(W, nbits=nbits, group_size=gs, axis=axis, round_zero=(nbits == 4), return_trace=True)
        pk = oracle.BIT_TO_PACKING[nbits]
        a, b = oracle.UNPACK[pk](Wq)[:rows].astype(int), oracle.UNPACK[pk](Wq_c)[:rows].astype(int)
        assert np.array_equal(s, meta_c["scale"].ravel()), case
        if heavy:
            assert abs(int(info[0]) - tr_c["iters"]) <= 1 and (a != b).mean() <= 2e-3 and np.abs(a - b).max() <= 1, case
        else:
            assert int(info[0]) == tr_c["iters"], case
            assert np.array_equal(a, b), case
            exact += 1
    assert exact >= 8


@pytest.mark.parametrize("nbits,gs,shape,axis", [(4, 64, (32, 256), 1), (2, 32, (16, 128), 1), (4, 64, (64, 48), 0), (3, 64, (25, 128), 1)])
def test_emulated_sharded_quantise_hooks_reproduce_the_one_call_path(emu, nbits, gs, shape, axis):
    """hqq_b200_quantize_shard_begin / _finish (the early stop taken from error sums the caller may all-reduce): with the shard's own
    sums and element count they must reproduce hqq_b200_quantize bit for bit; two 'ranks' that each hold half the rows and add their
    sums get the unsharded iteration count."""
    rng = np.random.default_rng(nbits * 7 + gs)
    W = (rng.standard_normal(shape) * 0.02).astype(np.float32)
    ref = quantize(emu, W, F32, nbits, gs, 1, axis=axis)
    emu.hqq_b200_quantize_shard_begin.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int64] + [ctypes.c_int] * 4 + \
        [ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    emu.hqq_b200_quantize_shard_finish.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int64] + [ctypes.c_int] * 4 + \
        [ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 6 + [ctypes.c_size_t, ctypes.c_void_p]

    def shard(Wp):
        N, K = Wp.shape
        Wd = aligned(Wp.shape, np.float32); Wd[...] = Wp
        nb = emu.hqq_b200_quantize_workspace_bytes(N, K, gs, nbits, axis, 20)
        ws = aligned((nb,), np.uint8)
        sums = aligned((20,), np.float64)
        rc = emu.hqq_b200_quantize_shard_begin(P(Wd), F32, N, K, gs, nbits, axis, int(nbits == 4), 0.7, 10.0, 20, P(sums), P(ws), nb, None)
        assert rc == 0, emu.hqq_b200_last_error()
        return Wd, ws, nb, sums

    def finish(Wd, ws, nb, sums, total):
        N, K = Wd.shape
        G = N * K // gs
        R, C = (G, gs) if axis == 1 else (gs, G)
        prow = -(-R // 10) if nbits == 3 else R // (8 // nbits)
        Wq = aligned((prow, C), np.int32 if nbits == 3 else np.uint8)
        s, z, info, err = aligned((G,), np.float32), aligned((G,), np.float32), aligned((4,), np.int32), aligned((20,), np.float32)
        rc = emu.hqq_b200_quantize_shard_finish(P(Wd), F32, N, K, gs, nbits, axis, int(nbits == 4), 0.7, 10.0, 20, P(sums), total, P(Wq), P(s), P(z),
                                                P(info), P(err), P(ws), nb, None)
        assert rc == 0, emu.hqq_b200_last_error()
        return Wq, s, z, info, err

    Wd, ws, nb, sums = shard(W)
    got = finish(Wd, ws, nb, sums, W.size)
    for x, y, what in zip(ref[:5], got, ("W_q", "scale", "zero", "info", "errors")):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), what
    if axis == 1 and nbits != 3:  # two ranks, half the rows each: global sums -> the unsharded stop
        h = shape[0] // 2
        a, b = shard(W[:h]), shard(W[h:])
        tot = aligned((20,), np.float64); tot[...] = a[3] + b[3]
        ia = finish(a[0], a[1], a[2], tot, W.size)[3]
        ib = finish(b[0], b[1], b[2], tot, W.size)[3]
        assert int(ia[0]) == int(ib[0]) == int(ref[3][0])


# ---------------------------------------------------------------------------------------------------------------------------------
# Decode glue kernels (csrc/decode_glue.cu, harness): the same source on the emulator against numpy restatements of the framework
# ops they replace.  (The cluster argmax is not emulated: DSMEM.)
def _f16(a):
    return np.asarray(a, dtype=np.float32).astype(np.float16)


def _rms_ref(h, delta, w, eps):
    """h = fl16(h + delta); y = fl16(fl16(h * rsqrt(mean(h^2) + eps)) * w), all in fp16 like `h = h + o; F.rms_norm(h, w)`"""
    x = h.astype(np.float32) if delta is None else (h.astype(np.float32) + delta.astype(np.float32)).astype(np.float16).astype(np.float32)
    inv = 1.0 / np.sqrt((x.astype(np.float64) ** 2).mean(axis=-1, keepdims=True) + eps)
    y = ((x * inv).astype(np.float16).astype(np.float32) * w.astype(np.float32)).astype(np.float16)
    return x.astype(np.float16), y


def test_emulated_add_rmsnorm_rows_and_silu_mul(emu):
    rng = np.random.default_rng(21)
    for rows, H in ((1, 4096), (5, 1024), (3, 8192), (2, 200)):
        h = aligned((rows, H), np.float16); d = aligned((rows, H), np.float16); w = aligned((H,), np.float16); y = aligned((rows, H), np.float16)
        h[...] = _f16(rng.standard_normal((rows, H))); d[...] = _f16(rng.standard_normal((rows, H))); w[...] = _f16(rng.random(H) + 0.5)
        for delta in (d, None):
            hh = aligned((rows, H), np.float16); hh[...] = h
            rc = emu.hqq_b200_glue_add_rmsnorm_rows(P(hh), P(delta), P(w), P(y), rows, H, ctypes.c_float(1e-5), F16, None)
            assert rc == 0, emu.hqq_b200_last_error()
            h_ref, y_ref = _rms_ref(h, delta, w, 1e-5)
            assert np.array_equal(hh, h_ref), (rows, H)                       # the residual stream: exactly fl16(h + delta)
            assert np.abs(y.astype(np.float32) - y_ref.astype(np.float32)).max() <= 2 ** -8 * np.abs(y_ref.astype(np.float32)).max()
            if rows > 1:                                                      # a row does not depend on its batch-mates
                h1 = aligned((1, H), np.float16); h1[...] = h[1:2]; y1 = aligned((1, H), np.float16)
                d1 = None
                if delta is not None:
                    d1 = aligned((1, H), np.float16); d1[...] = d[1:2]
                assert emu.hqq_b200_glue_add_rmsnorm(P(h1), P(d1), P(w), P(y1), H, ctypes.c_float(1e-5), F16, None) == 0
                assert np.array_equal(y1[0], y[1]) and np.array_equal(h1[0], hh[1])
    n = 3 * 1792 + 5
    g = aligned((n,), np.float16); u = aligned((n,), np.float16); o = aligned((n,), np.float16)
    g[...] = _f16(rng.standard_normal(n) * 3); u[...] = _f16(rng.standard_normal(n))
    assert emu.hqq_b200_glue_silu_mul(P(g), P(u), P(o), n, F16, None) == 0
    gf = g.astype(np.float32)
    ref = ((gf / (1.0 + np.exp(-gf))).astype(np.float16).astype(np.float32) * u.astype(np.float32)).astype(np.float16)
    assert np.abs(o.astype(np.float32) - ref.astype(np.float32)).max() <= 2 ** -9 * max(1.0, np.abs(ref.astype(np.float32)).max())


def _rope(x, cos, sin):
    """x*cos + rotate_half(x)*sin with every product and the sum rounded to fp16 (the framework ops' rounding)"""
    half = x.shape[-1] // 2
    rot = np.concatenate([-x[..., half:], x[..., :half]], axis=-1)
    a = (x.astype(np.float32) * cos.astype(np.float32)).astype(np.float16).astype(np.float32)
    b = (rot.astype(np.float32) * sin.astype(np.float32)).astype(np.float16).astype(np.float32)
    return (a + b).astype(np.float16)


def test_emulated_rope_attention_one_sequence_and_lock_step_batch(emu):
    """RoPE + KV-cache append + one-token GQA attention: cache rows written exactly, output against softmax(q k^T / sqrt(d)) v in
    float64; the lock-step batch entry point equals the one-sequence one sequence by sequence."""
    rng = np.random.default_rng(22)
    hq, hkv, hd, L, B = 4, 2, 128, 96, 3
    inv = 1.0 / (500000.0 ** (np.arange(0, hd, 2, dtype=np.float64) / hd))
    fr = np.outer(np.arange(L, dtype=np.float64), inv)
    cos = aligned((L, hd), np.float16); sin = aligned((L, hd), np.float16)
    cos[...] = _f16(np.concatenate([np.cos(fr), np.cos(fr)], -1)); sin[...] = _f16(np.concatenate([np.sin(fr), np.sin(fr)], -1))
    kc0 = _f16(rng.standard_normal((B, hkv, L, hd))); vc0 = _f16(rng.standard_normal((B, hkv, L, hd)))
    for pos in (0, 1, 37, 64, 95):
        q = aligned((B, hq * hd), np.float16); k = aligned((B, hkv * hd), np.float16); v = aligned((B, hkv * hd), np.float16)
        q[...] = _f16(rng.standard_normal(q.shape)); k[...] = _f16(rng.standard_normal(k.shape)); v[...] = _f16(rng.standard_normal(v.shape))
        kc = aligned(kc0.shape, np.float16); vc = aligned(vc0.shape, np.float16); out = aligned((B, hq * hd), np.float16)
        kc[...] = kc0; vc[...] = vc0
        p = aligned((1,), np.int64); p[0] = pos
        rc = emu.hqq_b200_glue_rope_attn_decode_batch(P(q), P(k), P(v), P(cos), P(sin), P(kc), P(vc), P(p), P(out), hq, hkv, L, hd, B, F16, None)
        assert rc == 0, emu.hqq_b200_last_error()
        for b in range(B):
            qr = _rope(q[b].reshape(hq, hd), cos[pos], sin[pos]); kr = _rope(k[b].reshape(hkv, hd), cos[pos], sin[pos])
            kref, vref = kc0[b].copy(), vc0[b].copy()
            kref[:, pos] = kr; vref[:, pos] = v[b].reshape(hkv, hd)
            assert np.array_equal(kc[b], kref) and np.array_equal(vc[b], vref), (pos, b)
            for h in range(hq):
                g = h // (hq // hkv)
                s = (kref[g, :pos + 1].astype(np.float64) @ qr[h].astype(np.float64)) / np.sqrt(hd)
                w = np.exp(s - s.max()); w /= w.sum()
                ref = w @ vref[g, :pos + 1].astype(np.float64)
                got = out[b, h * hd:(h + 1) * hd].astype(np.float64)
                assert np.abs(got - ref).max() <= 4e-3 * max(1.0, np.abs(ref).max()), (pos, b, h)
            # the one-sequence entry point on sequence b alone: bit-identical
            q1 = aligned((1, hq * hd), np.float16); k1 = aligned((1, hkv * hd), np.float16); v1 = aligned((1, hkv * hd), np.float16)
            q1[...] = q[b:b + 1]; k1[...] = k[b:b + 1]; v1[...] = v[b:b + 1]
            kc1 = aligned(kc0[b].shape, np.float16); vc1 = aligned(vc0[b].shape, np.float16); o1 = aligned((1, hq * hd), np.float16)
            kc1[...] = kc0[b]; vc1[...] = vc0[b]
            assert emu.hqq_b200_glue_rope_attn_decode(P(q1), P(k1), P(v1), P(cos), P(sin), P(kc1), P(vc1), P(p), P(o1), hq, hkv, L, hd, F16, None) == 0
            assert np.array_equal(o1[0], out[b]) and np.array_equal(kc1, kc[b]) and np.array_equal(vc1, vc[b]), (pos, b)


def test_emulated_add_rmsnorm_of_tagged_tensor_parallel_partials(emu):
    """hqq_b200_glue_add_rmsnorm_tp: the residual delta is the fp32 sum of `tp` tagged partial vectors {tag16 : value16} in this
    rank's exchange buffer (rounded once), the step counter is bumped; words of another exchange (other parity) are not touched."""
    rng = np.random.default_rng(23)
    H, tp, nb = 1024, 4, 3
    for step, x_index in ((0, 3), (5, 3), (6, 3)):
        ex = step * nb + x_index
        parts = _f16(rng.standard_normal((tp, H)))
        buf = aligned((2, tp, H), np.uint32)
        buf[...] = 0xFFFFFFFF
        buf[ex & 1] = (np.uint32(ex & 0xFFFF) << np.uint32(16)) | parts.view(np.uint16).astype(np.uint32)
        h = aligned((1, H), np.float16); w = aligned((H,), np.float16); y = aligned((1, H), np.float16)
        h0 = _f16(rng.standard_normal((1, H))); h[...] = h0; w[...] = _f16(rng.random(H) + 0.5)
        ctr = aligned((1,), np.int32); ctr[0] = step
        rc = emu.hqq_b200_glue_add_rmsnorm_tp(P(h), P(buf), P(ctr), x_index, nb, tp, P(w), P(y), H, ctypes.c_float(1e-5), F16, None)
        assert rc == 0, emu.hqq_b200_last_error()
        delta = parts.astype(np.float32).sum(axis=0, dtype=np.float32).astype(np.float16)   # fp32 sum in rank order, one rounding
        # (rank order matters in fp32: replay it exactly)
        acc = np.zeros(H, dtype=np.float32)
        for r in range(tp):
            acc = (acc + parts[r].astype(np.float32)).astype(np.float32)
        delta = acc.astype(np.float16)
        h_ref, y_ref = _rms_ref(h0, delta.reshape(1, H), w, 1e-5)
        assert np.array_equal(h, h_ref)
        assert np.abs(y.astype(np.float32) - y_ref.astype(np.float32)).max() <= 2 ** -8 * np.abs(y_ref.astype(np.float32)).max()
        assert int(ctr[0]) == step + 1
        assert np.all(buf[(ex & 1) ^ 1] == 0xFFFFFFFF)
