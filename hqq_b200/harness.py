"""Llama-shaped decode harness (SURVEY.md 8 f-2) -- the caller of HQQLinear.forward used by bench.py.

A random-init Llama-3-8B-*shaped* stack (no checkpoint is needed or loaded): every block linear
(q,k,v,o,gate,up,down -- the tags of hqq/models/hf/llama.py:12-21) is an ``HQQLinear`` quantised on the GPU by
this package; embeddings / lm_head / norms stay fp16 like the reference (hqq/models/base.py:43).  One decode
step = one token through all blocks with a static KV cache, captured once in a CUDA graph (the reference's
HFGenerator does the same with torch.compile + manual capture, hqq/utils/generation_hf.py:362-469; there is no
torch.compile here).  The non-linear glue (RMSNorm, RoPE, attention over the cache, SwiGLU) is plain PyTorch:
it is plumbing around the hot path, not part of it.

Tensor parallel (world_size > 1): q/k/v/gate/up are column-sharded (each rank quantises its own [N/tp, K]
shard -- slab packing cannot be sliced after the fact, SURVEY.md 7.7), o/down are row-sharded and end in ONE
all-reduce of the [1, hidden] activation, the only exchange step on the path (SURVEY.md 8e).
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from . import ops
from .core.quantize import BaseQuantizeConfig, HQQLinear


@dataclass
class LlamaShape:
    hidden: int = 4096
    inter: int = 14336
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int = 8
    vocab: int = 128256
    rope_theta: float = 500000.0
    rms_eps: float = 1e-5

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_heads


LLAMA3_8B = LlamaShape()
LLAMA3_70B = LlamaShape(hidden=8192, inter=28672, n_layers=80, n_heads=64, n_kv_heads=8)
TINY = LlamaShape(hidden=512, inter=1024, n_layers=2, n_heads=8, n_kv_heads=2, vocab=1024)


def shard_dims(shape: LlamaShape, tp: int):
    """Per-rank sizes of the sharded projections (pure host logic, unit-tested on CPU)."""
    if shape.n_heads % tp or shape.n_kv_heads % tp or shape.inter % tp:
        raise ValueError(f"tp={tp} must divide heads ({shape.n_heads}), kv heads ({shape.n_kv_heads}) and inter ({shape.inter})")
    hd = shape.head_dim
    return {"q": (shape.n_heads // tp * hd, shape.hidden), "k": (shape.n_kv_heads // tp * hd, shape.hidden),
            "v": (shape.n_kv_heads // tp * hd, shape.hidden), "o": (shape.hidden, shape.n_heads // tp * hd),
            "gate": (shape.inter // tp, shape.hidden), "up": (shape.inter // tp, shape.hidden),
            "down": (shape.hidden, shape.inter // tp)}


class DecodeModel:
    def __init__(self, shape: LlamaShape = LLAMA3_8B, nbits: int = 4, group_size: int = 64, dtype=torch.float16,
                 device="cuda", cache_len: int = 256, tp: int = 1, rank: int = 0, seed: int = 0, process_group=None,
                 n_layers: int | None = None, fused=5, tp_mode: str | None = None, batch: int = 1, shard_from_full: bool = False):
        self.shape, self.dtype, self.device = shape, dtype, torch.device(device)
        # batch > 1 (BASELINE configs[4], bs = 32): `batch` sequences decode in lock-step at the same position; the linears then
        # run the small-M kernel (M = batch <= 32; the wgmma kernel from 17 sequences on large matrices) between the batched glue
        # kernels -- the one-token kernels and their NVLink exchange are M = 1 only, so tensor-parallel partials are summed by NCCL
        self.batch = int(batch)
        if self.batch < 1:
            raise ValueError("batch must be >= 1")
        if self.batch > 1 and fused:
            fused = True  # the 8-launch path with the batched glue kernels; the one-token kernels (fused=5) and their exchange are M = 1 only
        self.fused = fused
        import os
        # "p2p": the row-parallel partials meet through tagged words over NVLink peer memory inside the kernels (default);
        # "nccl": NCCL all-reduce between the kernels (the correctness reference for the fused exchange, tools/tp_check.py)
        self.tp_mode = tp_mode or os.environ.get("HQQ_B200_TP_MODE", "p2p")
        if self.tp_mode not in ("p2p", "nccl"):
            raise ValueError(f"tp_mode must be 'p2p' or 'nccl' (got {self.tp_mode!r})")
        self.nbits, self.group_size = nbits, group_size
        self.tp, self.rank, self.pg = tp, rank, process_group
        self.cache_len = cache_len
        self.n_layers = n_layers if n_layers is not None else shape.n_layers
        dims = shard_dims(shape, tp)
        cfg = BaseQuantizeConfig(nbits=nbits, group_size=group_size, axis=1)
        g = torch.Generator(device=self.device)
        g.manual_seed(seed * 1000 + rank)
        gshared = torch.Generator(device=self.device)
        gshared.manual_seed(seed)

        def rnd(n, k, gen):
            return (torch.randn(n, k, device=self.device, generator=gen, dtype=torch.float32) * 0.02).to(dtype)

        self.embed = rnd(shape.vocab, shape.hidden, gshared)
        # lm_head stays fp16 like the reference (hqq/models/base.py:43); under tensor parallelism it is sharded by vocabulary:
        # every rank streams 1/tp of the rows and the argmax candidates meet in one 8-byte all-reduce (round 1 streamed the
        # full 1.05 GB head on every rank: 68 % of a rank's bytes at tp = 8)
        if shape.vocab % tp:
            raise ValueError(f"tp={tp} must divide the vocabulary ({shape.vocab})")
        self.vocab_shard = shape.vocab // tp
        head = rnd(shape.vocab, shape.hidden, gshared)
        self.lm_head = head[rank * self.vocab_shard:(rank + 1) * self.vocab_shard].clone() if tp > 1 else head
        del head
        self.final_norm = torch.ones(shape.hidden, device=self.device, dtype=dtype)
        self.blocks = []
        self.quantized_weights = 0
        # shard_from_full: every rank draws the FULL matrices from the shared generator, quantises them unsharded and cuts its shard out
        # of the quantised tensors (models/tp.py) -- the tensor-parallel model then computes the very function of the one-GPU model
        # (same levels, scales, zeros), which per-shard quantisation of per-rank random weights (the default, cheaper) does not
        full_dims = shard_dims(shape, 1)
        par = {"q": "column", "k": "column", "v": "column", "gate": "column", "up": "column", "o": "row", "down": "row"}
        for _ in range(self.n_layers):
            blk = {}
            for name, (n, k) in dims.items():
                if shard_from_full and tp > 1:
                    from .models.tp import shard_hqq_linear
                    fn, fk = full_dims[name]
                    full = HQQLinear.from_weights(rnd(fn, fk, gshared), None, cfg, compute_dtype=dtype, device=str(self.device))
                    blk[name] = shard_hqq_linear(full, tp, rank, par[name])
                    del full
                else:
                    blk[name] = HQQLinear.from_weights(rnd(n, k, gshared if shard_from_full else g), None, cfg, compute_dtype=dtype,
                                                       device=str(self.device))
                self.quantized_weights += n * k
            blk["norm1"] = torch.ones(shape.hidden, device=self.device, dtype=dtype)
            blk["norm2"] = torch.ones(shape.hidden, device=self.device, dtype=dtype)
            hkv = shape.n_kv_heads // tp
            blk["k_cache"] = torch.zeros(self.batch, hkv, cache_len, shape.head_dim, device=self.device, dtype=dtype)
            blk["v_cache"] = torch.zeros(self.batch, hkv, cache_len, shape.head_dim, device=self.device, dtype=dtype)
            self.blocks.append(blk)
        hd = shape.head_dim
        inv = 1.0 / (shape.rope_theta ** (torch.arange(0, hd, 2, device=self.device, dtype=torch.float32) / hd))
        t = torch.arange(cache_len, device=self.device, dtype=torch.float32)
        fr = torch.outer(t, inv)
        self.cos = torch.cat([fr.cos(), fr.cos()], dim=-1).to(dtype)  # [cache_len, hd]
        self.sin = torch.cat([fr.sin(), fr.sin()], dim=-1).to(dtype)
        self.arange = torch.arange(cache_len, device=self.device)
        # static I/O for graph capture
        self.tok = torch.zeros(self.batch, dtype=torch.long, device=self.device)
        self.pos = torch.zeros(1, dtype=torch.long, device=self.device)
        self.next_tok = torch.zeros(self.batch, dtype=torch.long, device=self.device)
        self.graph = None

    # bytes one decode step must read from HBM (SURVEY.md 8d): packed weights + meta + fp16 lm_head row-major
    def bytes_per_token(self, nbits=None, group_size=None) -> float:
        nbits = self.nbits if nbits is None else nbits
        group_size = self.group_size if group_size is None else group_size
        esize = torch.empty((), dtype=self.dtype).element_size()
        store = {8: 1.0, 4: 0.5, 3: 0.4, 2: 0.25, 1: 0.125}[int(nbits)]  # bytes per weight as packed (3-bit: 10 fields per int32)
        meta = 2 * esize / group_size                                       # scale + zero in the compute dtype
        return self.quantized_weights * (store + meta) + self.lm_head.numel() * esize

    @staticmethod
    def _multi(x, layers):
        outs = ops.linear_fwd_multi(x, layers)
        if outs is None:
            outs = [l(x) for l in layers]
        return outs

    def _rope(self, x, cos, sin):
        hd = x.shape[-1]
        x1, x2 = x[..., : hd // 2], x[..., hd // 2:]
        return x * cos + torch.cat((-x2, x1), dim=-1) * sin

    def step(self):
        """One token per sequence: reads self.tok [batch] / self.pos, writes self.next_tok and advances self.pos (all on device)."""
        s = self.shape
        B = self.batch
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        h = self.embed.index_select(0, self.tok)  # [B, hidden]
        cos = self.cos.index_select(0, self.pos).view(1, 1, hd)
        sin = self.sin.index_select(0, self.pos).view(1, 1, hd)
        mask = (self.arange <= self.pos).view(1, 1, 1, self.cache_len)
        for blk in self.blocks:
            x = F.rms_norm(h, (s.hidden,), blk["norm1"], s.rms_eps)
            q, k, v = self._multi(x, (blk["q"], blk["k"], blk["v"]))  # one launch: the three matrices share x
            q, k, v = q.view(B, hq, hd), k.view(B, hkv, hd), v.view(B, hkv, hd)
            q = self._rope(q, cos, sin)
            k = self._rope(k, cos, sin)
            blk["k_cache"].index_copy_(2, self.pos, k.view(B, hkv, 1, hd))
            blk["v_cache"].index_copy_(2, self.pos, v.view(B, hkv, 1, hd))
            a = F.scaled_dot_product_attention(q.view(B, hq, 1, hd), blk["k_cache"], blk["v_cache"], attn_mask=mask, enable_gqa=True)
            o = blk["o"](a.reshape(B, hq * hd))
            if self.tp > 1:
                torch.distributed.all_reduce(o, group=self.pg)
            h = h + o
            x = F.rms_norm(h, (s.hidden,), blk["norm2"], s.rms_eps)
            gate, up = self._multi(x, (blk["gate"], blk["up"]))
            y = blk["down"](F.silu(gate) * up)
            if self.tp > 1:
                torch.distributed.all_reduce(y, group=self.pg)
            h = h + y
        h = F.rms_norm(h, (s.hidden,), self.final_norm, s.rms_eps)
        logits = torch.matmul(h, self.lm_head.t())
        if self.tp > 1:  # vocabulary shards: the global maximum, then the lowest global index that attains it (two small all-reduces)
            val, idx = torch.max(logits.float(), dim=-1)
            gmax = val.clone()
            torch.distributed.all_reduce(gmax, op=torch.distributed.ReduceOp.MAX, group=self.pg)
            cand = torch.where(val == gmax, idx + self.rank * self.vocab_shard, torch.full_like(idx, s.vocab))
            torch.distributed.all_reduce(cand, op=torch.distributed.ReduceOp.MIN, group=self.pg)
            self.next_tok.copy_(cand)
        else:
            self.next_tok.copy_(torch.argmax(logits, dim=-1))
        self.pos.add_(1).remainder_(self.cache_len)

    def _head(self, lib, x, code, st):
        """Final projection + greedy pick inside the captured step: fp16 lm_head through the library GEMV (it is not an HQQ
        layer), then our argmax kernel; with tp > 1 each rank covers its vocabulary shard and the MAX of the ranks' 8-byte
        {value : index} keys picks the winner -- exchanged inside the argmax launch over peer-mapped memory ("p2p"), or by one
        NCCL all-reduce ("nccl")."""
        from ._lib import check, ptr
        b = self._bufs
        torch.matmul(x, self.lm_head.t(), out=b["logits"])
        if self.batch > 1:  # a row per sequence: framework ops (with tp > 1: the global maximum, then the lowest index that attains it)
            if self.tp == 1:
                self.next_tok.copy_(torch.argmax(b["logits"], dim=-1))
                return
            val, idx = torch.max(b["logits"].float(), dim=-1)
            gmax = val.clone()
            torch.distributed.all_reduce(gmax, op=torch.distributed.ReduceOp.MAX, group=self.pg)
            cand = torch.where(val == gmax, idx + self.rank * self.vocab_shard, torch.full_like(idx, self.shape.vocab))
            torch.distributed.all_reduce(cand, op=torch.distributed.ReduceOp.MIN, group=self.pg)
            self.next_tok.copy_(cand)
            return
        if self.tp == 1:
            check(lib.hqq_b200_glue_argmax(ptr(b["logits"]), self.vocab_shard, ptr(self.next_tok), code, st))
            return
        if self.fused == 5 and self.tp_mode == "p2p" and os.environ.get("HQQ_B200_HEAD_EXCHANGE", "p2p") != "nccl":  # (env: diagnosis only)
            # the keys meet in peer-mapped memory inside the argmax launch
            check(lib.hqq_b200_glue_argmax_tp(ptr(b["logits"]), self.vocab_shard, self.rank * self.vocab_shard, self._tp_keys, self.tp, self.rank,
                                              self._xstep.data_ptr(), ptr(self.next_tok), code, st))
            return
        check(lib.hqq_b200_glue_argmax_key(ptr(b["logits"]), self.vocab_shard, self.rank * self.vocab_shard, ptr(b["key"]), code, st))
        torch.distributed.all_reduce(b["key"], op=torch.distributed.ReduceOp.MAX, group=self.pg)
        torch.bitwise_and(b["key"], 0xFFFFFFFF, out=b["key"])
        self.next_tok.copy_(0xFFFFFFFF - b["key"])

    def _lin(self, x, layers, outs):
        """Matrices that share the activation x [B, K]: ONE launch of the small-M kernel when the router gives it all of them,
        else one routed call per matrix (from 17 rows on, matrices above 2^24 weights take the wgmma kernel, csrc/linear.cu)."""
        if ops.linear_fwd_multi(x, layers, outs) is not None:
            return
        for l, y in zip(layers, outs):
            m = l.meta
            store_bits = {"8bit_u8": 8, "4bit_u8": 4, "3bit_32": 3, "2bit_u8": 2, "1bit_u8": 1}[m["packing"]]
            if ops.linear_fwd(x, l.W_q, m["scale"], m["zero"], l.bias, int(m["shape"][0]), int(m["shape"][1]), m["group_size"], store_bits, m["axis"],
                              out=y) is None:
                raise RuntimeError("hqq_b200: no fused forward for this layer; use fused=False")

    def step_fused(self):
        """Same token step with the package's glue kernels (8 launches per block): add+RMSNorm, fused q/k/v, RoPE+cache+
        attention, o, add+RMSNorm, fused gate/up, SiLU*mul, down.  With tensor parallelism every rank runs the same launches
        on its shard (heads / inter split tp ways) and the two row-parallel outputs are summed with one all-reduce each."""
        from ._lib import DTYPE_CODE, check, load, ptr, stream_ptr
        lib, s = load(), self.shape
        st = stream_ptr(self.device)
        code = DTYPE_CODE[self.dtype]
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        inter = s.inter // self.tp
        b = self._bufs
        B = self.batch
        torch.index_select(self.embed, 0, self.tok, out=b["h"])  # [B, hidden]
        delta = None
        norm = lambda d, w: check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(b["h"]), ptr(d), ptr(w), ptr(b["x"]), B, s.hidden, s.rms_eps, code, st))
        for blk in self.blocks:
            norm(delta, blk["norm1"])
            self._lin(b["x"], (blk["q"], blk["k"], blk["v"]), [b["q"], b["k"], b["v"]])
            check(lib.hqq_b200_glue_rope_attn_decode_batch(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                           ptr(blk["v_cache"]), ptr(self.pos), ptr(b["a"]), hq, hkv, self.cache_len, hd, B, code, st))
            self._lin(b["a"], (blk["o"],), [b["o"]])
            if self.tp > 1:
                torch.distributed.all_reduce(b["o"], group=self.pg)
            norm(b["o"], blk["norm2"])
            self._lin(b["x"], (blk["gate"], blk["up"]), [b["gate"], b["up"]])
            check(lib.hqq_b200_glue_silu_mul(ptr(b["gate"]), ptr(b["up"]), ptr(b["act"]), B * inter, code, st))
            self._lin(b["act"], (blk["down"],), [b["down"]])
            if self.tp > 1:
                torch.distributed.all_reduce(b["down"], group=self.pg)
            delta = b["down"]
        norm(delta, self.final_norm)
        self._head(lib, b["x"], code, st)
        self.pos.add_(1).remainder_(self.cache_len)

    def _setup_exchange(self):
        """Buffers of tagged 32-bit words {tag16 : value16} through which the one-token kernels hand activations to each other
        (`hqq_b200_decode_linear_fwd_desc`): o / down partials [2 parities][tp][hidden] in peer-mapped symmetric memory, so the
        scatter + reduce IS the tensor-parallel all-reduce.  The step counter the tags derive from lives in local memory."""
        import ctypes
        s, tp, dev = self.shape, self.tp, self.device
        slot_bytes = 2 * tp * s.hidden * 4
        key_bytes = 2 * tp * 8  # argmax keys of the vocabulary-sharded lm_head, uint64 [2 parities][tp] (hqq_b200_glue_argmax_tp)
        if tp > 1:
            import torch.distributed as dist
            import torch.distributed._symmetric_memory as symm
            buf = symm.empty(2 * slot_bytes + key_bytes, dtype=torch.uint8, device=dev)
            buf.fill_(0xFF)  # tag 0xFFFF is only reached after 65535 exchanges; by then every word has been overwritten
            hdl = symm.rendezvous(buf, self.pg if self.pg is not None else dist.group.WORLD)
            ptrs = [int(p) for p in hdl.buffer_ptrs]
            self._xhdl = hdl
        else:
            buf = torch.full((2 * slot_bytes + key_bytes,), 0xFF, dtype=torch.uint8, device=dev)
            ptrs = [buf.data_ptr()]
        self._xbuf = buf
        self._xstep = torch.zeros(1, dtype=torch.int32, device=dev)
        VP = ctypes.c_void_p * tp
        self._tp_keep = [VP(*[p + slot * slot_bytes for p in ptrs]) for slot in range(2)]
        self._tp_local = [ptrs[self.rank] + slot * slot_bytes for slot in range(2)]
        self._tp_keys = VP(*[p + 2 * slot_bytes for p in ptrs])
        torch.cuda.synchronize(dev)
        if tp > 1:
            dist.barrier()

    def _tpx(self, block, **kw):
        d = {"tp": self.tp, "rank": self.rank, "step_ctr": self._xstep.data_ptr(), "x_index": block + 1, "x_per_step": len(self.blocks)}
        d.update(kw)
        return d

    def step_fused5(self):
        """Five launches per block: [add+RMSNorm -> q/k/v], RoPE+cache+attention, o, [add+RMSNorm -> gate/up -> SiLU*mul], down; the
        bracketed prologues / epilogue run inside the fused linears.  With tp > 1 and tp_mode "p2p" the o / down partials travel as
        tagged words over NVLink peer memory from the producing kernel's epilogue into the consuming kernel's prologue (the
        all-reduce is fused into both); tp_mode "nccl" puts an NCCL all-reduce between the kernels instead."""
        from ._lib import DTYPE_CODE, check, load, ptr, stream_ptr
        lib, s = load(), self.shape
        st = stream_ptr(self.device)
        code = DTYPE_CODE[self.dtype]
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        b = self._bufs
        h_cur, h_nxt = b["h"], b["h2"]
        torch.index_select(self.embed, 0, self.tok, out=h_cur)
        delta = None
        ok = True
        p2p = self.tp > 1 and self.tp_mode == "p2p"
        nb = len(self.blocks)
        pair = self.nbits < 8  # SiLU(gate) * up in the gate/up launch's epilogue (4/2/1-bit): computed once, not by each of down's CTAs
        if p2p:
            o_sc, d_sc = self._tp_keep            # scatter targets (every rank's buffer) for o / down
            o_loc, d_loc = self._tp_local         # this rank's buffers
        for bi, blk in enumerate(self.blocks):
            # [residual add + RMSNorm] -> q/k/v; p2p: the delta is the sum of the ranks' down-proj partials of block bi-1
            ok &= ops.decode_linear_fwd(h_cur, (blk["q"], blk["k"], blk["v"]), [b["q"], b["k"], b["v"]], 1, None if p2p else delta, blk["norm1"], h_nxt,
                                        s.rms_eps, tpx=(self._tpx(bi - 1, red_data=d_loc) if (p2p and bi > 0) else None))
            h_cur, h_nxt = h_nxt, h_cur
            check(lib.hqq_b200_glue_rope_attn_decode(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                     ptr(blk["v_cache"]), ptr(self.pos), ptr(b["a"]), hq, hkv, self.cache_len, hd, code, st))
            ok &= ops.decode_linear_fwd(b["a"], (blk["o"],), [b["o"]], tpx=self._tpx(bi, peer_data=o_sc) if p2p else None)
            if self.tp > 1 and not p2p:
                torch.distributed.all_reduce(b["o"], group=self.pg)
            gu_tpx = self._tpx(bi, red_data=o_loc) if p2p else None
            o_delta = None if p2p else b["o"]
            if pair:  # act = silu(gate) * up leaves the gate/up launch's epilogue; down takes it as is
                ok &= ops.decode_linear_fwd(h_cur, (blk["gate"], blk["up"]), [b["act"], b["up"]], 1 | ops.YOP_SILU_MUL_PAIR, o_delta, blk["norm2"],
                                            h_nxt, s.rms_eps, tpx=gu_tpx)
                h_cur, h_nxt = h_nxt, h_cur
                ok &= ops.decode_linear_fwd(b["act"], (blk["down"],), [b["down"]], tpx=self._tpx(bi, peer_data=d_sc) if p2p else None)
            else:
                ok &= ops.decode_linear_fwd(h_cur, (blk["gate"], blk["up"]), [b["gate"], b["up"]], 1, o_delta, blk["norm2"], h_nxt, s.rms_eps, tpx=gu_tpx)
                h_cur, h_nxt = h_nxt, h_cur
                ok &= ops.decode_linear_fwd(b["gate"], (blk["down"],), [b["down"]], 2, b["up"], tpx=self._tpx(bi, peer_data=d_sc) if p2p else None)
            if self.tp > 1 and not p2p:
                torch.distributed.all_reduce(b["down"], group=self.pg)
            delta = b["down"]
        if not ok:
            raise RuntimeError("hqq_b200: this model shape is outside the fused M=1 decode kernel; use fused=False or step_fused")
        if p2p:
            check(lib.hqq_b200_glue_add_rmsnorm_tp(ptr(h_cur), d_loc, self._xstep.data_ptr(), nb, nb, self.tp, ptr(self.final_norm),
                                                   ptr(b["x"]), s.hidden, s.rms_eps, code, st))
        else:
            check(lib.hqq_b200_glue_add_rmsnorm(ptr(h_cur), ptr(delta), ptr(self.final_norm), ptr(b["x"]), s.hidden, s.rms_eps, code, st))
        self._head(lib, b["x"], code, st)
        self.pos.add_(1).remainder_(self.cache_len)

    def _alloc_bufs(self):
        s, dev, dt = self.shape, self.device, self.dtype
        z = lambda n: torch.zeros(self.batch, n, device=dev, dtype=dt)
        tp = self.tp
        self._bufs = {"h": z(s.hidden), "h2": z(s.hidden), "x": z(s.hidden), "q": z(s.n_heads // tp * s.head_dim), "k": z(s.n_kv_heads // tp * s.head_dim),
                      "v": z(s.n_kv_heads // tp * s.head_dim), "a": z(s.n_heads // tp * s.head_dim), "o": z(s.hidden),
                      "gate": z(s.inter // tp), "up": z(s.inter // tp), "act": z(s.inter // tp), "down": z(s.hidden), "logits": z(self.vocab_shard),
                      "key": torch.zeros(1, dtype=torch.long, device=dev)}

    def capture(self, warmup: int = 3):
        """Warm up on a side stream, then capture one decode step into a CUDA graph."""
        fused = self.fused
        if fused and not hasattr(self, "_bufs"):
            self._alloc_bufs()
        if fused and self.fused == 5 and self.tp_mode == "p2p" and self.tp > 1 and not hasattr(self, "_xbuf"):
            self._setup_exchange()  # needs symmetric (peer-mapped) memory; ask for tp_mode="nccl" explicitly where that is not available
        step = (self.step_fused5 if self.fused == 5 else self.step_fused) if fused else self.step
        st = torch.cuda.Stream(device=self.device)
        st.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(st), torch.no_grad():
            for _ in range(warmup):
                step()
        torch.cuda.current_stream(self.device).wait_stream(st)
        torch.cuda.synchronize(self.device)
        self.pos.zero_()
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            step()
        return self.graph

    def reset_state(self, token: int = 1):
        """Position 0, empty KV caches, `token` as the first input: the state every token-stream comparison starts from."""
        self.tok.fill_(token)
        self.pos.zero_()
        for blk in self.blocks:
            blk["k_cache"].zero_()
            blk["v_cache"].zero_()
        if hasattr(self, "_bufs"):
            for t in self._bufs.values():
                t.zero_()

    def decode(self, feed_back: bool = True):
        """Replay one step; with feed_back the produced token becomes the next input (device-side copy)."""
        self.graph.replay()
        if feed_back:
            self.tok.copy_(self.next_tok)


# ---------------------------------------------------------------------------------------------- quantise-only sharding (SURVEY 8e)
def assign_layers(sizes, world: int):
    """Quantisation shards by layer with no collective (every linear depends only on its own weights, quantize.py:76-180):
    size-balanced assignment of layer indices to ranks -- largest first, each to the least-loaded rank (ties -> lowest rank),
    deterministic so every rank computes the same plan without talking.  Returns one index list per rank."""
    order = sorted(range(len(sizes)), key=lambda i: (-sizes[i], i))
    load = [0] * world
    plan = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda k: (load[k], k))
        plan[r].append(i)
        load[r] += sizes[i]
    return [sorted(p) for p in plan]
