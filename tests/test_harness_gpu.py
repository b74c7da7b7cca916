"""GPU: the decode harness (SURVEY.md 8 f-2) -- glue kernels vs the same ops in PyTorch, and the captured graph."""
import pytest
import torch
import torch.nn.functional as F

from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_glue_kernels_match_torch_ops(dt):
    lib = load()
    st = stream_ptr(DEV)
    code = DTYPE_CODE[dt]
    torch.manual_seed(0)
    H = 4096
    h = torch.randn(1, H, device=DEV).to(dt); d = torch.randn(1, H, device=DEV).to(dt); w = torch.rand(H, device=DEV).to(dt)
    h2 = h.clone(); y = torch.empty_like(h)
    check(lib.hqq_b200_glue_add_rmsnorm(ptr(h2), ptr(d), ptr(w), ptr(y), H, 1e-5, code, st))
    ref_h = h + d
    assert torch.equal(h2, ref_h)
    ref = F.rms_norm(ref_h, (H,), w, 1e-5)
    assert torch.allclose(y.float(), ref.float(), rtol=2e-2, atol=2e-2)
    g = torch.randn(1, 14336, device=DEV).to(dt); u = torch.randn(1, 14336, device=DEV).to(dt); o = torch.empty_like(g)
    check(lib.hqq_b200_glue_silu_mul(ptr(g), ptr(u), ptr(o), 14336, code, st))
    assert torch.allclose(o.float(), (F.silu(g) * u).float(), rtol=2e-2, atol=2e-2)
    lg = torch.randn(1, 128256, device=DEV).to(dt); out = torch.zeros(1, dtype=torch.long, device=DEV)
    check(lib.hqq_b200_glue_argmax(ptr(lg), 128256, ptr(out), code, st))
    assert int(out) == int(torch.argmax(lg.float(), dim=-1))
    for n, hot in ((5000, (4097, 77)), (13, (12,)), (8 * 8192 + 3, (8 * 8192 + 2, 8 * 8192 + 1))):  # ties -> first index; ragged tails
        lg = torch.zeros(1, n, device=DEV).to(dt)
        for i in hot:
            lg[0, i] = 3.0
        check(lib.hqq_b200_glue_argmax(ptr(lg), n, ptr(out), code, st))
        assert int(out) == min(hot), (n, int(out))


def _argmax_key(value: float, index: int, tag: int) -> int:
    """The 64-bit key hqq_b200_glue_argmax_tp exchanges (include/hqq_b200.h): ordered(value) >> 1 in the high word with the 12-bit
    tag in bits 32..43, 0xFFFFFFFF - index in the low word."""
    import struct
    u = struct.unpack("<I", struct.pack("<f", value))[0]
    ord_ = (~u & 0xFFFFFFFF) if (u & 0x80000000) else (u | 0x80000000)
    hi = ((ord_ >> 1) & ~0xFFF) | (tag & 0xFFF)
    return (hi << 32) | (0xFFFFFFFF - index)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_argmax_with_key_exchange_in_the_launch(dt):
    """hqq_b200_glue_argmax_tp on ONE GPU standing in for rank 0 of 2: both key areas are the same buffer and rank 1's key of the
    step is planted there beforehand.  The winner is the larger value, the lower index on equal values, whatever the sign; the
    key of an older step (another tag) in the slot is not taken for this step's."""
    import ctypes
    lib = load()
    st, code = stream_ptr(DEV), DTYPE_CODE[dt]
    torch.manual_seed(5)
    n, tp = 16032, 2
    VP = ctypes.c_void_p * tp
    out = torch.zeros(1, dtype=torch.long, device=DEV)
    for step, (local_top, peer_val, peer_idx) in enumerate(((3.0, 2.5, n + 7), (3.0, 3.5, n + 7), (3.0, 3.0, n + 900), (-2.0, -1.5, 2 * n - 1),
                                                            (-1.0, -1.5, n), (0.0, -0.5, n + 1)), start=1):
        lg = (torch.full((1, n), -4.0, device=DEV) - torch.rand(1, n, device=DEV)).to(dt)
        lg[0, 4321] = local_top
        lg[0, 9000] = local_top  # tie inside the shard: first index
        keys = torch.full((2 * tp,), -1, dtype=torch.long, device=DEV)  # 0xFF bytes, as the harness initialises the area
        ctr = torch.tensor([step], dtype=torch.int32, device=DEV)
        par = step & 1
        keys[par * tp + 1] = _argmax_key(peer_val, peer_idx, step)
        keys[(1 - par) * tp + 1] = _argmax_key(100.0, 5, step + 1)  # the other parity holds a key of another step: never read
        peers = VP(keys.data_ptr(), keys.data_ptr())
        check(lib.hqq_b200_glue_argmax_tp(ptr(lg), n, 0, peers, tp, 0, ctr.data_ptr(), ptr(out), code, st))
        torch.cuda.synchronize()
        want = peer_idx if peer_val > local_top else 4321
        assert int(out) == want, (step, int(out), want)
        assert int(keys[par * tp + 0]) == _argmax_key(local_top, 4321, step)  # what rank 0 published


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_rope_attention_kernel(dt):
    lib = load()
    st, code = stream_ptr(DEV), DTYPE_CODE[dt]
    torch.manual_seed(1)
    hq, hkv, hd, L = 8, 2, 128, 512
    m = harness.DecodeModel(harness.LlamaShape(hidden=hq * hd, inter=1024, n_layers=0, n_heads=hq, n_kv_heads=hkv, vocab=256), dtype=dt, device=DEV,
                            cache_len=L)
    kc = torch.randn(hkv, L, hd, device=DEV).to(dt); vc = torch.randn(hkv, L, hd, device=DEV).to(dt)
    for pos in (0, 1, 37, 63, 64, 200, 511):
        q = torch.randn(1, hq * hd, device=DEV).to(dt); k = torch.randn(1, hkv * hd, device=DEV).to(dt); v = torch.randn(1, hkv * hd, device=DEV).to(dt)
        kc1, vc1 = kc.clone(), vc.clone()
        p = torch.tensor([pos], device=DEV)
        out = torch.empty(1, hq * hd, device=DEV, dtype=dt)
        check(lib.hqq_b200_glue_rope_attn_decode(ptr(q), ptr(k), ptr(v), ptr(m.cos), ptr(m.sin), ptr(kc1), ptr(vc1), ptr(p), ptr(out), hq, hkv, L, hd, code, st))
        cos, sin = m.cos[pos].view(1, 1, hd), m.sin[pos].view(1, 1, hd)
        qr, kr = m._rope(q.view(1, hq, hd), cos, sin), m._rope(k.view(1, hkv, hd), cos, sin)
        kc2, vc2 = kc.clone(), vc.clone()
        kc2[:, pos] = kr[0]; vc2[:, pos] = v.view(hkv, hd)
        assert torch.equal(kc1, kc2) and torch.equal(vc1, vc2)
        mask = (torch.arange(L, device=DEV) <= pos).view(1, 1, 1, L)
        ref = F.scaled_dot_product_attention(qr.view(1, hq, 1, hd).float(), kc2[None].float(), vc2[None].float(), attn_mask=mask, enable_gqa=True)
        assert torch.allclose(out.float().view(hq, hd), ref.view(hq, hd), rtol=3e-2, atol=3e-2), pos


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nbits,N", [(4, 1024), (4, 1048), (2, 512), (1, 256)])
def test_paired_silu_mul_epilogue_is_bit_identical(dt, nbits, N):
    """x_op | HQQ_YOP_SILU_MUL_PAIR: y[0] = silu(gate) * up out of ONE launch == the two plain products + the glue kernel."""
    from hqq_b200 import ops
    from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear
    torch.manual_seed(nbits + N)
    K = 1024
    cfg = BaseQuantizeConfig(nbits=nbits, group_size=64, axis=1)
    gate, up = (HQQLinear.from_weights((torch.randn(N, K, device=DEV) * 0.05).to(dt), None, cfg, compute_dtype=dt, device=DEV) for _ in range(2))
    x = torch.randn(1, K, device=DEV).to(dt)
    g, u, act = (torch.empty(1, N, device=DEV, dtype=dt) for _ in range(3))
    assert ops.decode_linear_fwd(x, (gate, up), [g, u])
    ref = torch.empty_like(g)
    check(load().hqq_b200_glue_silu_mul(ptr(g), ptr(u), ptr(ref), N, DTYPE_CODE[dt], stream_ptr(DEV)))
    u2 = torch.full_like(u, 7.0)
    assert ops.decode_linear_fwd(x, (gate, up), [act, u2], ops.YOP_SILU_MUL_PAIR)
    assert torch.equal(act, ref)
    assert bool((u2 == 7.0).all())  # y[1] is not written
    # with the add + RMSNorm prologue in front (the MLP launch of the decode step)
    h, w, hout = torch.randn(1, K, device=DEV).to(dt), torch.rand(K, device=DEV).to(dt), torch.empty(1, K, device=DEV, dtype=dt)
    assert ops.decode_linear_fwd(x, (gate, up), [g, u], 1, h, w, hout, 1e-5)
    check(load().hqq_b200_glue_silu_mul(ptr(g), ptr(u), ptr(ref), N, DTYPE_CODE[dt], stream_ptr(DEV)))
    assert ops.decode_linear_fwd(x, (gate, up), [act, u2], 1 | ops.YOP_SILU_MUL_PAIR, h, w, hout, 1e-5)
    assert torch.equal(act, ref)


def test_ring_and_register_meta_paths_of_the_one_token_kernel_agree():
    """K % 512 == 0 with 16-byte aligned scale/zero rows takes the shipped kernel (scale/zero on the cp.async ring); a view whose meta
    rows start 8 bytes off takes the register-load instantiation of the same kernel.  Same bits."""
    from hqq_b200 import ops
    from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear
    for dt in (torch.float16, torch.bfloat16):
        for nbits in (4, 2, 1):
            torch.manual_seed(5 + nbits)
            lin = HQQLinear.from_weights((torch.randn(512, 1024, device=DEV) * 0.05).to(dt), None, BaseQuantizeConfig(nbits=nbits, group_size=64, axis=1),
                                         compute_dtype=dt, device=DEV)
            x = torch.randn(1, 1024, device=DEV).to(dt)
            y0, y1 = (torch.empty(1, 512, device=DEV, dtype=dt) for _ in range(2))
            assert ops.decode_linear_fwd(x, (lin,), [y0])
            # same values, scale / zero shifted by 4 elements (8 bytes): the ring's aligned 16-byte copies are not legal there
            s, z = lin.meta["scale"], lin.meta["zero"]
            for name, t in (("scale", s), ("zero", z)):
                buf = torch.empty(t.numel() + 4, device=DEV, dtype=t.dtype)
                buf[4:].copy_(t.view(-1))
                lin.meta[name] = buf[4:].view(t.shape)
            assert lin.meta["scale"].data_ptr() % 16 == 8
            assert ops.decode_linear_fwd(x, (lin,), [y1])
            torch.cuda.synchronize()
            assert torch.equal(y0, y1), (dt, nbits)


def test_paired_epilogue_rejects_what_it_cannot_pair():
    from hqq_b200 import ops
    from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear
    mk = lambda n, b: HQQLinear.from_weights((torch.randn(n, 512, device=DEV) * 0.05).half(), None, BaseQuantizeConfig(nbits=b, group_size=64, axis=1),
                                             compute_dtype=torch.float16, device=DEV)
    x = torch.randn(1, 512, device=DEV).half()
    o = lambda n: torch.empty(1, n, device=DEV, dtype=torch.float16)
    with pytest.raises(Exception):  # unequal N
        ops.decode_linear_fwd(x, (mk(256, 4), mk(512, 4)), [o(256), o(512)], ops.YOP_SILU_MUL_PAIR)
    assert not ops.decode_linear_fwd(x, (mk(256, 8), mk(256, 8)), [o(256), o(256)], ops.YOP_SILU_MUL_PAIR)  # 8-bit: unsupported -> caller falls back


def test_decode_graph_fused_equals_framework_ops():
    """A tiny 2-block model: the captured fused step (8 launches/block) and the PyTorch-op step produce the same tokens."""
    torch.manual_seed(0)
    shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
    models = []
    for f, m in ((5, "p2p"), (5, "nccl"), (True, None), (False, None)):
        models.append(harness.DecodeModel(shape, dtype=torch.float16, device=DEV, cache_len=32, fused=f, seed=3, tp_mode=m))
    toks = []
    for m in models:
        m.capture()
        m.tok.fill_(5); m.pos.zero_()
        for blk in m.blocks:
            blk["k_cache"].zero_(); blk["v_cache"].zero_()
        t = []
        for _ in range(12):
            m.decode()
            t.append(int(m.next_tok))
        toks.append(t)
    t5c, t5, t8, tref = toks
    assert t5c == t5, (t5c, t5)  # tp = 1: the two exchange modes are the same launches
    assert t5 == t8, (t5, t8)  # the in-kernel prologues round exactly like the stand-alone glue kernels
    agree = sum(int(x == y) for x, y in zip(t8, tref))
    assert agree >= 10, (t8, tref)  # fp16 reorderings may flip a near-tie late in the sequence, never the early tokens
    assert t8[:4] == tref[:4]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_batched_glue_kernels_equal_the_one_sequence_kernels_row_by_row(dt):
    """hqq_b200_glue_add_rmsnorm_rows / hqq_b200_glue_rope_attn_decode_batch (lock-step batch, one CTA per sequence / per head and
    sequence) produce, row by row, exactly what the one-sequence entry points produce."""
    lib = load()
    st, code = stream_ptr(DEV), DTYPE_CODE[dt]
    torch.manual_seed(11)
    B, H = 5, 4096
    h = torch.randn(B, H, device=DEV).to(dt); d = torch.randn(B, H, device=DEV).to(dt); w = torch.rand(H, device=DEV).to(dt)
    for delta in (d, None):
        hb, yb = h.clone(), torch.empty_like(h)
        check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(hb), ptr(delta), ptr(w), ptr(yb), B, H, 1e-5, code, st))
        for r in range(B):
            h1, y1 = h[r:r + 1].clone(), torch.empty(1, H, device=DEV, dtype=dt)
            check(lib.hqq_b200_glue_add_rmsnorm(ptr(h1), ptr(None if delta is None else delta[r:r + 1].contiguous()), ptr(w), ptr(y1), H, 1e-5, code, st))
            assert torch.equal(hb[r:r + 1], h1) and torch.equal(yb[r:r + 1], y1), r
    hq, hkv, hd, L = 8, 2, 128, 96
    m = harness.DecodeModel(harness.LlamaShape(hidden=hq * hd, inter=1024, n_layers=0, n_heads=hq, n_kv_heads=hkv, vocab=256), dtype=dt, device=DEV,
                            cache_len=L)
    kc = torch.randn(B, hkv, L, hd, device=DEV).to(dt); vc = torch.randn(B, hkv, L, hd, device=DEV).to(dt)
    for pos in (0, 5, 64, 95):
        q = torch.randn(B, hq * hd, device=DEV).to(dt); k = torch.randn(B, hkv * hd, device=DEV).to(dt); v = torch.randn(B, hkv * hd, device=DEV).to(dt)
        p = torch.tensor([pos], device=DEV)
        kb, vb, ob = kc.clone(), vc.clone(), torch.empty(B, hq * hd, device=DEV, dtype=dt)
        check(lib.hqq_b200_glue_rope_attn_decode_batch(ptr(q), ptr(k), ptr(v), ptr(m.cos), ptr(m.sin), ptr(kb), ptr(vb), ptr(p), ptr(ob), hq, hkv, L, hd, B,
                                                       code, st))
        for r in range(B):
            k1, v1, o1 = kc[r].clone(), vc[r].clone(), torch.empty(1, hq * hd, device=DEV, dtype=dt)
            check(lib.hqq_b200_glue_rope_attn_decode(ptr(q[r:r + 1].contiguous()), ptr(k[r:r + 1].contiguous()), ptr(v[r:r + 1].contiguous()), ptr(m.cos),
                                                     ptr(m.sin), ptr(k1), ptr(v1), ptr(p), ptr(o1), hq, hkv, L, hd, code, st))
            assert torch.equal(kb[r], k1) and torch.equal(vb[r], v1) and torch.equal(ob[r:r + 1], o1), (pos, r)


@pytest.mark.parametrize("batch,shape", [(4, harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)),
                                         (32, harness.LlamaShape(hidden=4096, inter=14336, n_layers=1, n_heads=32, n_kv_heads=8, vocab=4096))])
def test_batched_decode_graph_fused_equals_framework_ops(batch, shape):
    """Lock-step batch: the captured step on the batched glue kernels (add+RMSNorm rows, RoPE+attention per sequence, SiLU*mul; the
    linears through `_lin`: small-M kernel, or the wgmma kernel for 17+ sequences on matrices above 2^24 weights -- the second
    case has such matrices) against the same step on framework ops, every sequence starting from its own token."""
    toks = []
    for f in (True, False):
        m = harness.DecodeModel(shape, dtype=torch.float16, device=DEV, cache_len=32, fused=f, seed=3, batch=batch)
        assert m.fused is f
        m.capture()
        m.reset_state(1)
        m.tok.copy_(torch.arange(3, 3 + batch, device=DEV))
        t = []
        for _ in range(8):
            m.decode()
            t.append(m.next_tok.clone())
        toks.append(torch.stack(t))  # [steps, batch]
        del m
    a, b = toks
    assert torch.equal(a[:2], b[:2]), (a[:2], b[:2])                 # the first tokens of every sequence agree ...
    assert (a == b).float().mean().item() >= 0.9, (a, b)             # ... later ones up to fp16 near-ties (different summation orders)
    assert len(set(a[0].tolist())) > 1                               # the sequences are really different


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (tools/tp_check.py exercises the fused NVLink exchange on a 2-GPU machine)")
def test_tensor_parallel_peer_exchange_matches_nccl():
    """TP=2: the all-reduce fused into the row-parallel kernels over peer memory produces the same tokens as NCCL all-reduce."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", "29541", os.path.join(root, "tools", "tp_check.py")], capture_output=True, text=True, timeout=300)
    assert "AGREE 16 of 16" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_quantisation_equals_shards_of_the_unsharded_quantisation():
    """SURVEY 8e row 2: every rank quantises its rows / groups with the early stop taken from all-reduced error sums
    (hqq_b200_quantize_shard_begin / _finish) and gets exactly the shard models/tp.py cuts out of the unsharded quantisation."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", "29543", os.path.join(root, "tools", "tp_quant_check.py")], capture_output=True, text=True, timeout=300)
    assert "SHARDED-QUANT ALL-IDENTICAL" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
