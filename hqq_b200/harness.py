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
    # None: plain RoPE frequencies.  {"rope_type": "llama3", ...}: the Llama-3.1 frequency scaling (transformers' "llama3" rope type)
    rope_scaling: dict | None = None

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_heads


LLAMA3_8B = LlamaShape()
LLAMA3_70B = LlamaShape(hidden=8192, inter=28672, n_layers=80, n_heads=64, n_kv_heads=8)
TINY = LlamaShape(hidden=512, inter=1024, n_layers=2, n_heads=8, n_kv_heads=2, vocab=1024)
# Llama-3.1 / 3.3 (128k context): the Llama-3 shapes with the llama3 RoPE scaling
LLAMA31_8B = LlamaShape(rope_scaling={"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                      "original_max_position_embeddings": 8192})

# Above this many cache positions the fused steps run the split-KV attention kernel (csrc/decode_glue.cu): the one-CTA-per-head
# kernel keeps a score per position in shared memory and stops here.  At or below it they run that kernel as before.
SINGLE_ATTN_MAX_LEN = 8192
LOGPROB_ROWS = 4096  # rows per hqq_b200_lm_logprob call in score(): 33 MB of tile partials at vocabulary 128256


def rope_inv_freq(shape: LlamaShape, device) -> torch.Tensor:
    """RoPE inverse frequencies [head_dim / 2] in fp32; with rope_scaling "llama3" scaled as transformers'
    `_compute_llama3_parameters` does it (same fp32 operations in the same order)."""
    hd = shape.head_dim
    inv = 1.0 / (shape.rope_theta ** (torch.arange(0, hd, 2, device=device, dtype=torch.float32) / hd))
    sc = shape.rope_scaling
    if sc is None:
        return inv
    if sc.get("rope_type") != "llama3":
        raise ValueError(f"unsupported rope_scaling {sc!r}: only rope_type 'llama3' is implemented")
    factor, lf, hf = float(sc["factor"]), float(sc["low_freq_factor"]), float(sc["high_freq_factor"])
    old = float(sc["original_max_position_embeddings"])
    low_wl, high_wl = old / lf, old / hf
    wavelen = 2 * math.pi / inv
    inv_l = torch.where(wavelen > low_wl, inv / factor, inv)
    smooth = (old / wavelen - lf) / (hf - lf)
    smoothed = (1 - smooth) * inv_l / factor + smooth * inv_l
    medium = ~(wavelen < high_wl) * ~(wavelen > low_wl)
    return torch.where(medium, smoothed, inv_l)


def rope_tables(shape: LlamaShape, cache_len: int, dtype, device):
    """cos / sin tables [cache_len, head_dim] in `dtype` (the glue kernels read them by position)."""
    inv = rope_inv_freq(shape, device)
    t = torch.arange(cache_len, device=device, dtype=torch.float32)
    fr = torch.outer(t, inv)
    return torch.cat([fr.cos(), fr.cos()], dim=-1).to(dtype), torch.cat([fr.sin(), fr.sin()], dim=-1).to(dtype)


def kv8_quantize_rows(x: torch.Tensor, group_size: int, bits: int = 8):
    """The 8-bit KV cache format on framework ops: rows x [..., 128] in T -> levels uint8 [..., 128] and scale, zero
    [..., 128 / group_size] in T.  HQQ's Quantizer.quantize(row, nbits=8, group_size, axis=1, optimize=False) (round_zero off, as for
    8-bit layers) in fp32 -- inverse scale reciprocal(max - min) * 255 (1 where max - min <= 1e-4, at most 2e4), zero -min * s,
    levels round(x * s + z) clamped to [0, 255] with the product and the sum rounded separately -- then scale = 1 / s and the zero
    cast to T.  The solver is not run: its early stop compares a mean over the whole tensor, so a row's levels would depend on
    which rows were quantised with it.  bits 4: the 4-bit cache, nbits=4 (15 in place of 255, group_size 32 or 64), each row's levels
    packed as the reference's 4bit_u8 packing of that row: uint8 [..., 64], byte d = q[d] << 4 | q[d + 64]."""
    maxv = float((1 << bits) - 1)
    shape = x.shape
    w = x.float().reshape(-1, group_size)
    mn, mx = w.amin(dim=1, keepdim=True), w.amax(dim=1, keepdim=True)
    denom = mx - mn
    s = torch.reciprocal(denom) * maxv
    s = torch.where(denom.abs() <= 1e-4, torch.ones_like(s), s)
    s = torch.clamp(s, max=2e4)
    z = -mn * s
    q = torch.clamp(torch.round(w * s + z), 0, maxv).to(torch.uint8).reshape(shape)
    if bits == 4:
        half = shape[-1] // 2
        q = (q[..., :half] << 4) | q[..., half:]
    meta = shape[:-1] + (shape[-1] // group_size,)
    return q, torch.reciprocal(s).to(x.dtype).reshape(meta), z.to(x.dtype).reshape(meta)


def kv8_dequantize(q: torch.Tensor, scale: torch.Tensor, zero: torch.Tensor, bits: int = 8) -> torch.Tensor:
    """Rows of the 8-bit KV cache back in T: (T(q) - zero) * scale with one rounding to T per operation (hqq_b200_dequantize,
    Quantizer.dequantize).  q [..., 128] uint8, scale / zero [..., 128 / group_size] in T.  bits 4: q [..., 64] packed as
    kv8_quantize_rows packs it, unpacked first."""
    if bits == 4:
        q = torch.cat([q >> 4, q & 15], dim=-1)
    ng = scale.shape[-1]
    qs = q.reshape(q.shape[:-1] + (ng, q.shape[-1] // ng)).to(scale.dtype)
    return ((qs - zero.unsqueeze(-1)) * scale.unsqueeze(-1)).reshape(q.shape)


_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)
_U32 = 0xFFFFFFFF


def _mulhilo32(a: torch.Tensor, m: int):
    """High and low 32-bit words of a * m, a int64 in [0, 2^32), m a 32-bit constant; exact in int64 through 16-bit limbs."""
    p0 = a * (m & 0xFFFF)                # < 2^48
    p1 = a * (m >> 16)                   # < 2^48
    s = ((p1 & 0xFFFF) << 16) + p0       # < 2^49
    return (p1 >> 16) + (s >> 32), s & _U32


def position_counter(pos: torch.Tensor, seq: torch.Tensor) -> torch.Tensor:
    """Counter words 2 and 3 of hqq_b200_glue_sample_pos for rows at positions pos of sequences seq (int64 [rows] each): int64
    [rows, 2] = (pos & 0xFFFFFFFF, 0x80000000 | (seq & 0x7FFFFFFF)), for philox_uniforms / sample_tokens with the row's slot as b."""
    return torch.stack((pos.to(torch.int64) & _U32, (seq.to(torch.int64) & 0x7FFFFFFF) | 0x80000000), dim=-1)


def philox_uniforms(n: int, rows: int, seed: int, counter, device=None) -> torch.Tensor:
    """The race's uniforms of hqq_b200_glue_sample on framework ops: u [rows, n] in float64, u[b, i] = ((x >> 9) + 0.5) * 2^-23 with x
    word i % 4 of Philox4x32-10 under key (seed & 0xFFFFFFFF, seed >> 32) and counter (i / 4, b, ctr & 0xFFFFFFFF, ctr >> 32).
    counter: a python int or an int64 tensor of one element (read on the device, so a captured graph sees it advance); or an int64
    tensor [rows, 2] of per-row counter words 2 and 3 (position_counter: hqq_b200_glue_sample_pos's keys, row b being slot b)."""
    if not torch.is_tensor(counter):
        counter = torch.tensor([int(counter)], dtype=torch.int64, device=device)
    device = counter.device
    nq = -(-n // 4)
    c0 = torch.arange(nq, dtype=torch.int64, device=device).view(1, nq).expand(rows, nq)
    c1 = torch.arange(rows, dtype=torch.int64, device=device).view(rows, 1).expand(rows, nq)
    if counter.dim() == 2:
        w = counter.to(torch.int64) & _U32
        c2, c3 = w[:, :1].expand(rows, nq), w[:, 1:].expand(rows, nq)
    else:
        ctr = counter.reshape(1, 1).to(torch.int64)
        c2, c3 = (ctr & _U32).expand(rows, nq), ((ctr >> 32) & _U32).expand(rows, nq)
    k0, k1 = int(seed) & _U32, (int(seed) >> 32) & _U32
    for r in range(10):
        if r:
            k0, k1 = (k0 + _PHILOX_W[0]) & _U32, (k1 + _PHILOX_W[1]) & _U32
        hi0, lo0 = _mulhilo32(c0, _PHILOX_M[0])
        hi1, lo1 = _mulhilo32(c2, _PHILOX_M[1])
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    x = torch.stack((c0, c1, c2, c3), dim=-1).reshape(rows, 4 * nq)[:, :n]
    return ((x >> 9).double() + 0.5) * 2.0 ** -23


def sample_tokens(logits: torch.Tensor, temperature: float, top_k: int, top_p: float, seed: int, counter) -> torch.Tensor:
    """hqq_b200_glue_sample restated on framework ops in float64 (the definition is in include/hqq_b200.h): logits [rows, n] in
    fp16 / bf16, row b sampled with Philox counter (., b, counter), counter as philox_uniforms takes it (per-row words 2 and 3
    restate hqq_b200_glue_sample_pos); returns int64 [rows].  temperature and top_p are taken at fp32
    precision, as the kernel receives them.  Top-k compares the 16-bit values as stored.  The reference generator's
    torch.where(logits < pivot, -inf, logits) on fp16(logits / T) can merge neighbouring values by that rounding; here they stay
    apart, so its keep set can be larger than ours at the pivot."""
    T = float(torch.tensor(temperature, dtype=torch.float32))
    P = float(torch.tensor(top_p, dtype=torch.float32))
    rows, n = logits.shape
    lv = logits.double()
    keep = torch.ones_like(lv, dtype=torch.bool)
    if 0 < top_k < n:
        keep = lv >= torch.topk(lv, top_k, dim=-1).values[:, -1:]
    if P < 1.0:
        w = torch.where(keep, torch.exp((lv - lv.amax(dim=-1, keepdim=True)) / T), torch.zeros_like(lv))
        vs, order = torch.sort(torch.where(keep, lv, torch.full_like(lv, -math.inf)), dim=-1, descending=True)
        cum = w.gather(1, order).cumsum(dim=-1)
        j = (cum < P * cum[:, -1:]).sum(dim=-1, keepdim=True).clamp(max=n - 1)
        keep = keep & (lv >= vs.gather(1, j))
    u = philox_uniforms(n, rows, seed, counter, logits.device)
    key = torch.where(keep, lv / T - torch.log(-torch.log(u)), torch.full_like(lv, -math.inf))
    return torch.argmax(key, dim=-1)


KV_PAGE = 64  # positions per page of a paged KV cache (csrc/decode_glue.cu kPage)


class PageAllocator:
    """Host bookkeeping of a paged KV cache (DecodeModel(kv_pages=N)), pure Python: no device access, so it is testable without a
    GPU.  Pages 0 .. N-1 are real, page N is the sink.  table[b][j] names the page that holds positions 64 j .. 64 j + 63 of slot b;
    every entry not backed by a real page points at the sink, so an entry is always a valid index.  A real page carries one reference
    per table entry that names it, and returns to the free list when the last one goes.  pos mirrors the device positions (every
    slot steps, a released one into the sink); active marks the slots whose steps get pages.

    Invariant: the entries past a slot's current page are the sink.  So a slot only writes into pages it entered fresh or copied,
    and a shared page is never written.  Each operation returns (writes, copies): table entries (b, j, page) to store on the device
    and pages (src, dst) to copy in every layer, copies first.  An operation that runs out of pages raises RuntimeError and leaves
    the state as it was."""

    def __init__(self, n_pages: int, batch: int, cache_len: int):
        if not (isinstance(n_pages, int) and n_pages >= 1):
            raise ValueError(f"kv_pages must be an int >= 1 (got {n_pages!r})")
        if cache_len % KV_PAGE:
            raise ValueError(f"a paged cache needs cache_len % {KV_PAGE} == 0 (got {cache_len})")
        self.n_pages, self.batch, self.cache_len = n_pages, batch, cache_len
        self.sink = n_pages
        self.entries = cache_len // KV_PAGE
        self.reset()

    def reset(self):
        """Every page free, every entry the sink, every slot active at position 0."""
        self.table = [[self.sink] * self.entries for _ in range(self.batch)]
        self.ref = [0] * self.n_pages
        self.free = list(range(self.n_pages - 1, -1, -1))  # pop() hands out the lowest free page
        self.pos = [0] * self.batch
        self.active = [True] * self.batch

    @property
    def free_pages(self) -> int:
        return len(self.free)

    def pages_of(self, b: int) -> int:
        return sum(p != self.sink for p in self.table[b])

    # ---- primitives: they record the device writes in w
    def _take(self):
        if not self.free:
            raise RuntimeError(f"paged KV cache: out of pages (all {self.n_pages} in use)")
        p = self.free.pop()
        self.ref[p] = 1
        return p

    def _drop(self, p):
        if p != self.sink:
            self.ref[p] -= 1
            if self.ref[p] == 0:
                self.free.append(p)

    def _set(self, w, b, j, p):
        self.table[b][j] = p
        w.append((b, j, p))

    def _clear(self, w, b, first=0):
        """Entries first.. of slot b back to the sink."""
        for j in range(first, self.entries):
            if self.table[b][j] != self.sink:
                self._drop(self.table[b][j])
                self._set(w, b, j, self.sink)

    def _atomic(self, fn):
        snap = ([r[:] for r in self.table], self.ref[:], self.free[:], self.pos[:], self.active[:])
        try:
            return fn()
        except (RuntimeError, ValueError):
            self.table, self.ref, self.free, self.pos, self.active = snap
            raise

    # ---- operations
    def step(self):
        """Pages for one decode step, then every position advances by one (mod cache_len).  An active slot about to write row p with
        p % 64 == 0 gets a fresh page for entry p / 64; at p == 0 (the wrap) its previous lap's pages are returned first."""
        edge = [b for b in range(self.batch) if self.active[b] and self.pos[b] % KV_PAGE == 0]

        def run():
            w = []
            for b in edge:  # every reference is given up before any page is taken
                if self.pos[b] == 0:
                    self._clear(w, b)
                else:
                    j = self.pos[b] // KV_PAGE
                    self._drop(self.table[b][j])
            for b in edge:
                self._set(w, b, self.pos[b] // KV_PAGE, self._take())
            return w, []
        ops = self._atomic(run) if edge else ([], [])
        self.pos = [(p + 1) % self.cache_len for p in self.pos]
        return ops

    def spec_window(self, k: int):
        """Pages for one speculative verify step (before it runs): an active slot writes rows pos .. pos + n - 1, n = min(k + 1,
        cache_len - pos).  Every entry the window enters at the page's first row gets a fresh page (the entry the window starts in
        mid-page is the slot's current page, backed already); at pos == 0 (the wrap) the previous lap's pages are returned first.
        Positions do not move: spec_advance does that once the accepted counts are known."""
        spans = {b: (self.pos[b], min(k + 1, self.cache_len - self.pos[b])) for b in range(self.batch) if self.active[b]}

        def run():
            w, fresh = [], []
            for b, (p, n) in spans.items():  # every reference is given up before any page is taken
                if p == 0:
                    self._clear(w, b)
                for j in range(p // KV_PAGE, (p + n - 1) // KV_PAGE + 1):
                    if j * KV_PAGE >= p:
                        self._drop(self.table[b][j])
                        fresh.append((b, j))
            for b, j in fresh:
                self._set(w, b, j, self._take())
            return w, []
        return self._atomic(run)

    def spec_advance(self, n_new):
        """After a verify step: every slot's position moves by its n_new[b] accepted tokens (mod cache_len), and an active slot's
        pages that lie wholly at or past its new position (they hold only rejected rows) go back to the pool.  Restores the
        invariant: entries past the page of the slot's last written row are the sink."""
        w = []
        for b in range(self.batch):
            self.pos[b] = (self.pos[b] + int(n_new[b])) % self.cache_len
            if self.active[b]:
                self._clear(w, b, -(-self.pos[b] // KV_PAGE))
        return w, []

    def prefill(self, spans):
        """Back the rows a prefill writes.  spans: {slot: (start, T)}, rows start .. start + T - 1.  A page the prompt enters at its
        first row gets a fresh page; the page it enters mid-page must be backed already and is copied first if shared.  Entries past
        the prompt's last page go back to the sink.  ValueError if positions [0, start) hold no pages."""
        for b, (start, _) in spans.items():
            if any(self.table[b][j] == self.sink for j in range(-(-start // KV_PAGE))):
                raise ValueError(f"slot {b}: positions [0, {start}) are not all backed by pages (released, or never written)")

        def run():
            w, copies, fresh = [], [], []
            for b, (start, T) in spans.items():
                first, last = start // KV_PAGE, (start + T - 1) // KV_PAGE
                self._clear(w, b, last + 1)
                for j in range(first, last + 1):
                    p = self.table[b][j]
                    if j * KV_PAGE >= start:
                        self._drop(p)
                        fresh.append((b, j))
                    elif self.ref[p] > 1:  # copy-on-write of the shared page the prompt continues
                        q = self._take()
                        copies.append((p, q))
                        self._drop(p)
                        self._set(w, b, j, q)
            for b, j in fresh:
                self._set(w, b, j, self._take())
            for b, (start, T) in spans.items():
                self.pos[b] = (start + T) % self.cache_len
                self.active[b] = True
            return w, copies
        return self._atomic(run)

    def release(self, b: int):
        """Slot b's pages back to the free list, its entries to the sink; it keeps stepping, into the sink, until a prefill or a
        fork targets it again."""
        w = []
        self._clear(w, b)
        self.active[b] = False
        return w, []

    def fork(self, src: int, dst: int):
        """dst continues src: dst is released, then shares src's full pages below pos[src] and gets a copy of the partial one."""
        if src == dst:
            raise ValueError("fork needs two different slots")
        if not self.active[src]:
            raise ValueError(f"slot {src} is released: nothing to fork")

        def run():
            w, copies = self.release(dst)
            p = self.pos[src]
            for j in range(p // KV_PAGE):
                pg = self.table[src][j]
                self.ref[pg] += 1
                self._set(w, dst, j, pg)
            if p % KV_PAGE:
                q = self._take()
                copies.append((self.table[src][p // KV_PAGE], q))
                self._set(w, dst, p // KV_PAGE, q)
            self.pos[dst] = p
            self.active[dst] = True
            return w, copies
        return self._atomic(run)


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
                 n_layers: int | None = None, fused=5, tp_mode: str | None = None, batch: int = 1, shard_from_full: bool = False,
                 kv_bits: int = 16, kv_group_size: int | None = None, do_sample: bool = False, temperature: float = 0.6, top_k: int = 5,
                 top_p: float = 1.0, sample_seed: int = 0, ragged: bool = False, kv_pages: int | None = None, spec_k: int | None = None,
                 sample_keys: str = "step"):
        self.shape, self.dtype, self.device = shape, dtype, torch.device(device)
        # do_sample: every token (decode steps, batch rows, the token prefill returns) is drawn by hqq_b200_glue_sample -- temperature,
        # top-k, top-p, then a Gumbel race on Philox numbers keyed by sample_seed and countered by _sample_ctr -- instead of the argmax.
        # The defaults are those of the reference's HFGenerator; like there, the parameters are fixed for the model's life.
        t32 = float(torch.tensor(float(temperature), dtype=torch.float32)) if isinstance(temperature, (int, float)) else math.nan
        if not (math.isfinite(t32) and t32 > 0):  # the kernel takes it as fp32
            raise ValueError(f"temperature must be finite and > 0 in fp32 (got {temperature!r})")
        if not (isinstance(top_k, int) and top_k >= 0):
            raise ValueError(f"top_k must be an int >= 0, 0 for off (got {top_k!r})")
        if not (isinstance(top_p, (int, float)) and 0 < float(torch.tensor(float(top_p), dtype=torch.float32)) <= 1 and top_p <= 1):
            raise ValueError(f"top_p must lie in (0, 1], 1 for off (got {top_p!r})")
        if not (isinstance(sample_seed, int) and 0 <= sample_seed < 2 ** 64):
            raise ValueError(f"sample_seed must be an int in [0, 2^64) (got {sample_seed!r})")
        self.do_sample, self.temperature, self.top_k, self.top_p, self.sample_seed = bool(do_sample), float(temperature), int(top_k), float(top_p), int(sample_seed)
        # sample_keys "position" (do_sample): the token drawn from the row at position p of slot b takes the Philox numbers keyed by
        # (b, p, seq[b]) (hqq_b200_glue_sample_pos), seq the slot's sequence number.  A sequence's token at a position then draws the
        # same numbers in decode(), prefill() and decode_spec(), and does not depend on when other slots were refilled; this is what
        # lets sampling and speculative decoding combine.  "step" (the default): the counter _sample_ctr, + 1 per sampling call.
        if sample_keys not in ("step", "position"):
            raise ValueError(f"sample_keys must be 'step' or 'position' (got {sample_keys!r})")
        if sample_keys == "position" and not self.do_sample:
            raise ValueError("sample_keys='position' needs do_sample=True")
        self.position_keys = sample_keys == "position"
        # kv_bits 8: every layer's K and V cache in HQQ's 8-bit format (kv8_quantize_rows), groups of kv_group_size along the head dim;
        # kv_bits 4: HQQ's 4-bit format, each row's levels packed by 4bit_u8 (kv8_quantize_rows(..., bits=4)), groups of 32 or 64.
        # kv_group_size defaults to 64 for the 8-bit cache; the 4-bit cache takes it explicitly: at 4 bits the group size is the
        # cache's accuracy / size trade-off (gs 32: 160 bytes per position and kv head, gs 64: 144), not a detail to default silently
        if kv_bits not in (16, 8, 4):
            raise ValueError(f"kv_bits must be 16, 8 or 4 (got {kv_bits!r})")
        if kv_group_size is None:
            if kv_bits == 4:
                raise ValueError("kv_bits=4 needs an explicit kv_group_size, 32 or 64")
            kv_group_size = 64
        if kv_bits == 4 and kv_group_size not in (32, 64):
            raise ValueError(f"kv_group_size must be 32 or 64 with kv_bits=4 (got {kv_group_size!r})")
        if kv_bits != 4 and kv_group_size not in (64, 128):
            raise ValueError(f"kv_group_size must be 64 or 128 (got {kv_group_size!r})")
        if kv_bits != 16 and shape.head_dim != 128:
            raise ValueError(f"kv_bits={kv_bits} needs head_dim 128")
        self.kv_bits, self.kv_group_size = int(kv_bits), int(kv_group_size)
        self._kvq = self.kv_bits != 16  # a quantised cache: levels plus scale and zero
        # batch > 1 (BASELINE configs[4], bs = 32): `batch` sequences decode in lock-step at the same position; the linears then
        # run the small-M kernel (M = batch <= 32; the wgmma kernel from 17 sequences on large matrices) between the batched glue
        # kernels -- the one-token kernels and their NVLink exchange are M = 1 only, so tensor-parallel partials are summed by NCCL
        self.batch = int(batch)
        if self.batch < 1:
            raise ValueError("batch must be >= 1")
        # ragged: every sequence sits at its own position (self.pos is int64 [batch]); prefill takes prompts of different lengths in
        # one packed pass and can refill one slot while the others keep their caches.  The decode steps run the _seqpos attention
        # kernels, prefill the _varlen ones; everything else is row-independent at M = batch already.
        self.ragged = bool(ragged)
        if self.ragged and self.batch > 256:
            raise ValueError("ragged batches hold at most 256 sequences")
        if self.kv_bits == 4 and self.batch > 256:  # the staging refill takes the batch as slots
            raise ValueError("kv_bits=4 holds at most 256 sequences")
        # kv_pages N (ragged only): every layer's cache is a pool of N + 1 pages [N + 1, n_kv, 64, 128] (page N the sink) and the
        # slots reach their rows through one shared device page_table [batch, cache_len / 64]; PageAllocator hands out the pages.
        # The kernels are the ragged ones' PAGED twins: a paged model computes the unpaged ragged model's bits.
        self.kv_pages = kv_pages
        if kv_pages is not None:
            if not self.ragged:
                raise ValueError("kv_pages needs ragged=True")
            self.pages = PageAllocator(kv_pages, self.batch, cache_len)
        # spec_k K (ragged): decode_spec() verifies the window [tok, d1 .. dK] of every slot in one captured pass and emits the
        # accepted drafts plus one target (include/hqq_b200.h states the rule); the drafts come from prompt lookup over the device
        # token history `hist` [batch, cache_len] or from the caller.  The targets are the rows' greedy picks, or with do_sample and
        # position keys their sampled tokens: for one-token drafts, accepting while draft == target is exact speculative sampling.
        self.spec_k = spec_k
        if spec_k is not None:
            if not self.ragged:
                raise ValueError("spec_k needs ragged=True")
            if do_sample and not self.position_keys:
                raise ValueError("spec_k verifies greedy targets: it cannot be combined with do_sample")
            if not (isinstance(spec_k, int) and 1 <= spec_k <= 7):
                raise ValueError(f"spec_k must be an int in [1, 7] (got {spec_k!r})")
        if (self.batch > 1 or self.ragged) and fused:
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
            cdt = torch.uint8 if self._kvq else dtype
            rows = (self.batch, hkv, cache_len) if kv_pages is None else (kv_pages + 1, hkv, KV_PAGE)
            width = shape.head_dim * self.kv_bits // 8 if self._kvq else shape.head_dim  # level bytes or elements a row
            blk["k_cache"] = torch.zeros(*rows, width, device=self.device, dtype=cdt)
            blk["v_cache"] = torch.zeros(*rows, width, device=self.device, dtype=cdt)
            if self._kvq:
                for name in ("k_scale", "k_zero", "v_scale", "v_zero"):
                    blk[name] = torch.zeros(*rows, shape.head_dim // kv_group_size, device=self.device, dtype=dtype)
            self.blocks.append(blk)
        self._kv8_stage = None  # kv_bits 8 / 4: dequantised fp16 / bf16 K and V for the prefill attention, allocated by the first fused prefill
        self.cos, self.sin = rope_tables(shape, cache_len, dtype, self.device)  # [cache_len, hd]
        self.arange = torch.arange(cache_len, device=self.device)
        # static I/O for graph capture
        self.tok = torch.zeros(self.batch, dtype=torch.long, device=self.device)
        self.pos = torch.zeros(self.batch if self.ragged else 1, dtype=torch.long, device=self.device)
        self._slot_idx = torch.arange(self.batch, device=self.device)
        self.next_tok = torch.zeros(self.batch, dtype=torch.long, device=self.device)
        self._sample_ctr = torch.zeros(1, dtype=torch.long, device=self.device)  # Philox counter: + 1 per sampled token
        # position keys: slot b's sequence number, + 1 when a prefill starts the slot at position 0, copied by fork()
        self.seq = torch.zeros(self.batch, dtype=torch.long, device=self.device) if self.position_keys else None
        if kv_pages is not None:
            self.page_table = torch.full((self.batch, cache_len // KV_PAGE), kv_pages, dtype=torch.int32, device=self.device)
        if spec_k is not None:  # hist[b][p] = the token fed at position p; the verify step's static I/O
            self.hist = torch.zeros(self.batch, cache_len, dtype=torch.int32, device=self.device)
            self._spec_drafts = torch.full((self.batch, spec_k), -1, dtype=torch.long, device=self.device)
            self._spec_targets = torch.zeros(self.batch * (spec_k + 1), dtype=torch.long, device=self.device)
            self._spec_tokens = torch.full((self.batch, spec_k + 1), -1, dtype=torch.long, device=self.device)
            self._spec_n_new = torch.zeros(self.batch, dtype=torch.long, device=self.device)
            self.spec_graph = None
            self.spec_logits = None  # [batch, K + 1, vocab / tp]: the last verify step's logits
        self.graph = None
        self.last_logits = None  # set by prefill(): logits of the last prompt position of each sequence

    @property
    def attn_kernel(self) -> str:
        """Attention kernel of the fused steps: "single" (one CTA per query head, cache_len <= 8192), "split" (split-KV) or
        "split_kv8" / "split_kv4" (split-KV over the 8-bit / 4-bit cache, at every cache_len)."""
        if self._kvq:
            return f"split_kv{self.kv_bits}"
        return "split" if self.cache_len > SINGLE_ATTN_MAX_LEN else "single"

    _CACHE_NAMES = ("k_cache", "v_cache", "k_scale", "k_zero", "v_scale", "v_zero")

    @property
    def free_pages(self) -> int:
        """kv_pages: the pages no slot holds."""
        return self.pages.free_pages

    def cache_view(self, blk) -> dict:
        """A layer's caches in the contiguous layout [batch, n_kv, cache_len, ...]: the tensors themselves, or with kv_pages a copy
        gathered through the page table (rows no page backs read the sink)."""
        names = [n for n in self._CACHE_NAMES if n in blk]
        if self.kv_pages is None:
            return {n: blk[n] for n in names}
        idx = self.page_table.long()
        B, E = idx.shape
        return {n: blk[n][idx].permute(0, 2, 1, 3, 4).reshape(B, blk[n].shape[1], E * KV_PAGE, blk[n].shape[3]) for n in names}

    def _apply_pages(self, ops):
        """A PageAllocator operation's result on the device, in stream order and without a sync: page copies in every layer, then
        the table entries (scalar fills)."""
        writes, copies = ops
        for src, dst in copies:
            for blk in self.blocks:
                for n in self._CACHE_NAMES:
                    if n in blk:
                        blk[n][dst].copy_(blk[n][src])
        for b, j, p in writes:
            self.page_table[b, j] = p

    def release(self, b: int):
        """kv_pages: slot b's pages go back to the pool and its table row to the sink.  The slot keeps stepping (all slots do), into
        the sink; its tokens mean nothing until a prefill or a fork targets it again.  The other slots are unaffected."""
        self._paged_only("release")
        self._apply_pages(self.pages.release(int(b)))

    def fork(self, src: int, dst: int):
        """kv_pages: slot dst continues slot src -- dst is released, then shares src's full pages below pos[src] (stored once) and
        gets a copy of the partial page in every layer; pos and tok (and with position keys seq) are copied.  Neither slot ever writes a shared page."""
        self._paged_only("fork")
        src, dst = int(src), int(dst)
        if not (0 <= src < self.batch and 0 <= dst < self.batch):
            raise ValueError(f"fork: slots must lie in [0, {self.batch})")
        self._apply_pages(self.pages.fork(src, dst))
        self.pos[dst].copy_(self.pos[src])
        self.tok[dst].copy_(self.tok[src])
        if self.seq is not None:
            self.seq[dst].copy_(self.seq[src])
        if self.spec_k is not None:
            self.hist[dst].copy_(self.hist[src])

    def _paged_only(self, what):
        if self.kv_pages is None:
            raise ValueError(f"{what} needs a paged KV cache (kv_pages)")

    def kv_cache_bytes(self) -> int:
        """Bytes of every layer's KV cache on this rank: fp16 / bf16 rows, or levels plus scale and zero with kv_bits 8 / 4 (with
        kv_pages: the page pools, sink included)."""
        names = ("k_cache", "v_cache", "k_scale", "k_zero", "v_scale", "v_zero")
        return sum(blk[n].numel() * blk[n].element_size() for blk in self.blocks for n in names if n in blk)

    def _attn_split(self, lib, blk, hq, hkv, code, st):
        from ._lib import check, ptr
        b = self._bufs
        paged = self.kv_pages is not None
        kvq = f"kv{self.kv_bits}"
        if paged and self._kvq:
            check(getattr(lib, f"hqq_b200_glue_rope_attn_decode_split_{kvq}_paged")(
                ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]), ptr(blk["k_scale"]), ptr(blk["k_zero"]),
                ptr(blk["v_cache"]), ptr(blk["v_scale"]), ptr(blk["v_zero"]), ptr(self.page_table), ptr(self.pos), ptr(b["a"]), ptr(b["attn_ws"]), hq,
                hkv, self.cache_len, self.shape.head_dim, self.kv_group_size, self.batch, self.kv_pages, code, st))
            return
        if paged:
            check(lib.hqq_b200_glue_rope_attn_decode_split_paged(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                                 ptr(blk["v_cache"]), ptr(self.page_table), ptr(self.pos), ptr(b["a"]), ptr(b["attn_ws"]), hq,
                                                                 hkv, self.cache_len, self.shape.head_dim, self.batch, self.kv_pages, code, st))
            return
        if self._kvq:
            fn = getattr(lib, f"hqq_b200_glue_rope_attn_decode_split_{kvq}" + ("_seqpos" if self.ragged else ""))
            check(fn(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                     ptr(blk["k_scale"]), ptr(blk["k_zero"]), ptr(blk["v_cache"]), ptr(blk["v_scale"]),
                     ptr(blk["v_zero"]), ptr(self.pos), ptr(b["a"]), ptr(b["attn_ws"]), hq, hkv, self.cache_len,
                     self.shape.head_dim, self.kv_group_size, self.batch, code, st))
            return
        fn = lib.hqq_b200_glue_rope_attn_decode_split_seqpos if self.ragged else lib.hqq_b200_glue_rope_attn_decode_split
        check(fn(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                 ptr(blk["v_cache"]), ptr(self.pos), ptr(b["a"]), ptr(b["attn_ws"]), hq, hkv, self.cache_len,
                 self.shape.head_dim, self.batch, code, st))

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
        self._hist_write()
        h = self.embed.index_select(0, self.tok)  # [B, hidden]
        if self.ragged:  # sequence b at position pos[b]: its own RoPE row and causal mask
            cos = self.cos.index_select(0, self.pos).view(B, 1, hd)
            sin = self.sin.index_select(0, self.pos).view(B, 1, hd)
            mask = (self.arange.view(1, -1) <= self.pos.view(B, 1)).view(B, 1, 1, self.cache_len)
        else:
            cos = self.cos.index_select(0, self.pos).view(1, 1, hd)
            sin = self.sin.index_select(0, self.pos).view(1, 1, hd)
            mask = (self.arange <= self.pos).view(1, 1, 1, self.cache_len)
        for blk in self.blocks:
            x = F.rms_norm(h, (s.hidden,), blk["norm1"], s.rms_eps)
            q, k, v = self._multi(x, (blk["q"], blk["k"], blk["v"]))  # one launch: the three matrices share x
            q, k, v = q.view(B, hq, hd), k.view(B, hkv, hd), v.view(B, hkv, hd)
            q = self._rope(q, cos, sin)
            k = self._rope(k, cos, sin)
            if self.ragged:  # row pos[b] of sequence b (kv_pages: through the page table)
                if self.kv_pages is None:
                    at = (self._slot_idx, slice(None), self.pos)
                else:
                    at = (self.page_table[self._slot_idx, self.pos // KV_PAGE].long(), slice(None), self.pos % KV_PAGE)
                for name, x in (("k", k), ("v", v.view(B, hkv, hd))):
                    if self._kvq:
                        lv, sc, ze = kv8_quantize_rows(x, self.kv_group_size, self.kv_bits)
                        for suffix, val in (("_cache", lv), ("_scale", sc), ("_zero", ze)):
                            blk[name + suffix][at] = val
                    else:
                        blk[name + "_cache"][at] = x
                cv = self.cache_view(blk)
                kc, vc = self._kv8_read(cv, self.cache_len) if self._kvq else (cv["k_cache"], cv["v_cache"])
            elif self._kvq:  # the rotated rows quantised into the cache; attention over the dequantised cache
                self._kv8_write(blk, k.view(B, hkv, 1, hd), v.view(B, hkv, 1, hd), self.pos)
                kc, vc = self._kv8_read(blk, self.cache_len)
            else:
                blk["k_cache"].index_copy_(2, self.pos, k.view(B, hkv, 1, hd))
                blk["v_cache"].index_copy_(2, self.pos, v.view(B, hkv, 1, hd))
                kc, vc = blk["k_cache"], blk["v_cache"]
            a = F.scaled_dot_product_attention(q.view(B, hq, 1, hd), kc, vc, attn_mask=mask, enable_gqa=True)
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
        if self.do_sample:
            self.next_tok.copy_(self._sample_ref(logits, self.pos.expand(B)))
            self._sample_ctr.add_(1)
        elif self.tp > 1:  # vocabulary shards: the global maximum, then the lowest global index that attains it (two small all-reduces)
            val, idx = torch.max(logits.float(), dim=-1)
            gmax = val.clone()
            torch.distributed.all_reduce(gmax, op=torch.distributed.ReduceOp.MAX, group=self.pg)
            cand = torch.where(val == gmax, idx + self.rank * self.vocab_shard, torch.full_like(idx, s.vocab))
            torch.distributed.all_reduce(cand, op=torch.distributed.ReduceOp.MIN, group=self.pg)
            self.next_tok.copy_(cand)
        else:
            self.next_tok.copy_(torch.argmax(logits, dim=-1))
        self.pos.add_(1).remainder_(self.cache_len)

    def _hist_write(self):
        """spec_k: a decode step records its input token in the prompt-lookup history, hist[b][pos[b]] = tok[b]."""
        if self.spec_k is not None:
            self.hist.scatter_(1, self.pos.view(-1, 1), self.tok.view(-1, 1).to(torch.int32))

    def _kv8_write(self, blk, k, v, idx):
        """kv_bits 8 / 4 on framework ops: rows k, v [batch, n_kv, n, 128] quantised into cache positions idx [n]."""
        for name, x in (("k", k), ("v", v)):
            lv, sc, ze = kv8_quantize_rows(x, self.kv_group_size, self.kv_bits)
            blk[name + "_cache"].index_copy_(2, idx, lv)
            blk[name + "_scale"].index_copy_(2, idx, sc)
            blk[name + "_zero"].index_copy_(2, idx, ze)

    def _kv8_read(self, blk, end):
        """kv_bits 8 / 4 on framework ops: the dequantised K and V cache rows [0, end)."""
        return tuple(kv8_dequantize(blk[n + "_cache"][:, :, :end], blk[n + "_scale"][:, :, :end], blk[n + "_zero"][:, :, :end], self.kv_bits) for n in ("k", "v"))

    def _sample_ref(self, logits, pos=None):
        """do_sample on framework ops (fused=False): sample_tokens on the full-vocabulary rows (under tensor parallelism every rank
        gathers the shards and draws the same tokens).  Row b is slot b; with position keys pos [rows] holds the rows' positions."""
        if self.tp > 1:
            g = torch.empty(self.tp * logits.shape[0], logits.shape[1], dtype=logits.dtype, device=logits.device)
            torch.distributed.all_gather_into_tensor(g, logits.contiguous(), group=self.pg)
            logits = g.view(self.tp, -1, self.vocab_shard).transpose(0, 1).reshape(-1, self.shape.vocab)
        ctr = position_counter(pos, self.seq) if self.position_keys else self._sample_ctr
        return sample_tokens(logits, self.temperature, self.top_k, self.top_p, self.sample_seed, ctr)

    def _sample_buffers(self, rows):
        """What _sample_rows needs for `rows` sequences: the all-gather target under tensor parallelism, and padded rows where the
        gathered layout or the vocabulary length does not give 16-byte aligned rows."""
        n, d = self.shape.vocab, {}
        if self.tp > 1:
            d["sample_gather"] = torch.zeros(self.tp * rows, self.vocab_shard, dtype=self.dtype, device=self.device)
        if n % 8 or (self.tp > 1 and rows > 1):
            d["sample_rows"] = torch.zeros(rows, -(-n // 8) * 8, dtype=self.dtype, device=self.device)
        return d

    def _sample_rows(self, logits, bufs):
        """Full-vocabulary rows for hqq_b200_glue_sample from this rank's logits [rows, vocab / tp]: with tp > 1 one NCCL all-gather
        of the shards (capturable), rearranged to [rows, vocab] when rows > 1; rows padded to a multiple of 8 elements when the
        vocabulary is not one (the kernel reads 16-byte vectors)."""
        B, n = logits.shape[0], self.shape.vocab
        if self.tp > 1:
            g = bufs["sample_gather"]
            torch.distributed.all_gather_into_tensor(g, logits, group=self.pg)
            if "sample_rows" not in bufs:
                return g.view(B, n)  # one row: the shards follow each other
            src = g.view(self.tp, B, self.vocab_shard).transpose(0, 1)  # [B, tp, vocab / tp]
        else:
            if "sample_rows" not in bufs:
                return logits
            src = logits.view(B, 1, n)
        rows = bufs["sample_rows"]
        rows[:, :n].view(B, self.tp, self.vocab_shard).copy_(src)
        return rows

    def _sample(self, lib, rows, out, code, st, pos=None, T=1):
        """One launch of hqq_b200_glue_sample over rows [B, >= vocab]: out[b] = the token of row b at the current _sample_ctr.  With
        position keys hqq_b200_glue_sample_pos instead: row r is slot r / T at position pos[r / T] + r % T (pos: device int64)."""
        from ._lib import check, ptr
        if self.position_keys:
            check(lib.hqq_b200_glue_sample_pos(ptr(rows), self.shape.vocab, rows.stride(0), rows.shape[0], self.temperature, self.top_k, self.top_p,
                                               self.sample_seed, T, ptr(pos), ptr(self.seq), ptr(out), code, st))
            return
        check(lib.hqq_b200_glue_sample(ptr(rows), self.shape.vocab, rows.stride(0), rows.shape[0], self.temperature, self.top_k, self.top_p,
                                       self.sample_seed, ptr(self._sample_ctr), ptr(out), code, st))

    def _step_pos(self):
        """Position keys in a captured step: the rows' positions, one per slot (a lock-step model's single position copied to every
        slot inside the step)."""
        if self.pos.numel() == self.batch:
            return self.pos
        p = self._bufs["sample_pos"]
        p.copy_(self.pos.expand(self.batch))
        return p

    def _head(self, lib, x, code, st):
        """Final projection + greedy pick inside the captured step: fp16 lm_head through the library GEMV (it is not an HQQ
        layer), then our argmax kernel; with tp > 1 each rank covers its vocabulary shard and the MAX of the ranks' 8-byte
        {value : index} keys picks the winner -- exchanged inside the argmax launch over peer-mapped memory ("p2p"), or by one
        NCCL all-reduce ("nccl").  do_sample: the sampling kernel on the full rows instead (with tp > 1 after one all-gather of the
        shards, so every rank draws the same token)."""
        from ._lib import check, ptr
        b = self._bufs
        torch.matmul(x, self.lm_head.t(), out=b["logits"])
        if self.do_sample:
            self._sample(lib, self._sample_rows(b["logits"], b), self.next_tok, code, st, pos=self._step_pos() if self.position_keys else None)
            return
        if self.batch > 1:  # a row per sequence: framework ops
            self.next_tok.copy_(self._greedy(b["logits"]))
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
        self._hist_write()
        torch.index_select(self.embed, 0, self.tok, out=b["h"])  # [B, hidden]
        delta = None
        norm = lambda d, w: check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(b["h"]), ptr(d), ptr(w), ptr(b["x"]), B, s.hidden, s.rms_eps, code, st))
        for blk in self.blocks:
            norm(delta, blk["norm1"])
            self._lin(b["x"], (blk["q"], blk["k"], blk["v"]), [b["q"], b["k"], b["v"]])
            if self.attn_kernel != "single":
                self._attn_split(lib, blk, hq, hkv, code, st)
            elif self.kv_pages is not None:
                check(lib.hqq_b200_glue_rope_attn_decode_batch_paged(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin),
                                                                     ptr(blk["k_cache"]), ptr(blk["v_cache"]), ptr(self.page_table), ptr(self.pos),
                                                                     ptr(b["a"]), hq, hkv, self.cache_len, hd, B, self.kv_pages, code, st))
            else:
                fn = lib.hqq_b200_glue_rope_attn_decode_batch_seqpos if self.ragged else lib.hqq_b200_glue_rope_attn_decode_batch
                check(fn(ptr(b["q"]), ptr(b["k"]), ptr(b["v"]), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                         ptr(blk["v_cache"]), ptr(self.pos), ptr(b["a"]), hq, hkv, self.cache_len, hd, B, code,
                         st))
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
        if self.do_sample:
            self._sample_ctr.add_(1)

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
            if self.attn_kernel != "single":
                self._attn_split(lib, blk, hq, hkv, code, st)
            else:
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
        if self.do_sample:
            self._sample_ctr.add_(1)

    def prefill(self, tokens: torch.Tensor, start: int = 0, chunk: int = 2048) -> torch.Tensor:
        """Take in a prompt: `tokens` [batch, T] (or [T] when batch is 1) at positions start .. start + T - 1 of every sequence.
        The prompt runs in chunks of at most `chunk` tokens (batch * chunk <= 65535, the row limit of the rows kernels); each
        chunk goes through every block, writing its rotated k and v into the caches.  Only the last position of each sequence
        goes through the final norm, the lm_head and the argmax (with do_sample: the sampling kernel at the current sample counter,
        which then advances by one; with position keys at the last prompt position, after a prefill from position 0 has added one
        to every slot's sequence number seq); self.last_logits [batch, vocab / tp] keeps those logits (this rank's vocabulary shard).  Afterwards self.pos = (start + T) mod cache_len -- the steps' own wrap, so a prompt that fills
        the cache leaves the next step at position 0 as a step at the last position does -- and self.tok [batch] holds the greedy
        (do_sample: the sampled) next token, which is returned: a captured decode step continues from there.

        fused (any value but False): the package's kernels -- add+RMSNorm rows, the routed q/k/v linears at M = batch * chunk,
        RoPE + cache append, causal GQA attention over the cache (csrc/decode_glue.cu), o, add+RMSNorm rows, gate/up, SiLU*mul,
        down.  fused=False: the same walk on framework ops (F.rms_norm, the layers, torch RoPE, F.scaled_dot_product_attention
        with a causal mask over the cache), the correctness reference as step() is for decode.  With tensor parallelism the two
        row-parallel outputs and the head's argmax keys meet in NCCL all-reduces; the peer-memory exchange of fused=5 decode and
        its step counter are not touched.

        kv_bits 8: the rows kernel quantises k and v into the 8-bit cache as the decode kernel does and writes their dequantisation
        into a staging pair [batch, n_kv, cache_len, 128] in T (allocated once, shared by all layers); staging rows [0, start of the
        chunk) are dequantised from the cache per layer and chunk (hqq_b200_dequantize), and the attention kernel reads the staging
        pair.  fused=False quantises into the cache and attends over its dequantisation.

        ragged: see _prefill_ragged (`tokens` is a list of per-slot prompts or None)."""
        return self._prefill(tokens, start, chunk)

    def score(self, prompts, start: int = 0, chunk: int = 2048):
        """prefill() with the same arguments, checks and resulting state (caches, pos, tok, last_logits, the sample counter, pages,
        hist), which also returns the prompt's log-probabilities: entry i is log p(prompt[i + 1] | prompt[0 .. i] and the cache rows
        before the prompt), fp32; the first prompt token is not scored.  Lock-step: a [batch, T - 1] tensor; ragged: one 1-D tensor
        of T_b - 1 entries per slot (None for slots without a prompt).

        After the last block of each chunk every row goes through the final norm (hqq_b200_glue_add_rmsnorm_rows on a copy of the
        residual stream) and the LSE head (hqq_b200_lm_logprob, blocks of at most LOGPROB_ROWS rows; the target of a row is the
        slot's next prompt token, -1 at its last position): log p = tgt - lse, and the logits never reach memory.  The last
        positions also go through prefill's own head, unchanged.  With tensor parallelism each rank's (lse, tgt) meet in one
        all_gather_into_tensor and are merged in rank order, so every rank returns the same values.  fused=False: torch.matmul
        logits, F.log_softmax in fp32 and a gather (the logits of all ranks gathered first) -- the reference."""
        logp = {}
        self._prefill(prompts, start, chunk, score=logp)
        return logp["out"]

    def _score_rows(self, h, delta, targets):
        """log p(targets | rows) fp32 [R] for the residual stream h, delta [R, hidden] after the last block; h is not modified.
        Rows whose target is -1 get an arbitrary value (the callers drop them)."""
        s, R = self.shape, h.shape[0]
        if not self.fused:
            x = F.rms_norm(h + delta, (s.hidden,), self.final_norm, s.rms_eps)
            logits = torch.matmul(x, self.lm_head.t())
            if self.tp > 1:
                g = torch.empty(self.tp, R, self.vocab_shard, dtype=logits.dtype, device=logits.device)
                torch.distributed.all_gather_into_tensor(g, logits.contiguous(), group=self.pg)
                logits = g.permute(1, 0, 2).reshape(R, -1)
            lp = F.log_softmax(logits.float(), dim=-1)
            return lp.gather(1, targets.clamp_min(0).view(-1, 1)).view(-1)
        from ._lib import DTYPE_CODE, check, load, ptr, stream_ptr
        lib, st, code = load(), stream_ptr(self.device), DTYPE_CODE[self.dtype]
        hs, x = h.clone(), torch.empty_like(h)
        check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(hs), ptr(delta), ptr(self.final_norm), ptr(x), R, s.hidden, s.rms_eps, code, st))
        n = self.vocab_shard
        lse = torch.empty(2, R, dtype=torch.float32, device=self.device)  # [lse; tgt]
        rows = min(R, LOGPROB_ROWS)
        ws = torch.empty(lib.hqq_b200_lm_logprob_workspace_bytes(rows, n), dtype=torch.uint8, device=self.device)
        for r0 in range(0, R, rows):
            m = min(rows, R - r0)
            check(lib.hqq_b200_lm_logprob(ptr(x[r0:]), ptr(self.lm_head), ptr(targets[r0:]), ptr(lse[0, r0:]), ptr(lse[1, r0:]), ptr(ws), m, n,
                                          s.hidden, self.rank * n, code, st))
        if self.tp > 1:  # lse = M + log(sum_r exp(lse_r - M)) in rank order; tgt is finite on the one rank whose shard holds it
            g = torch.empty(self.tp, 2, R, dtype=torch.float32, device=self.device)
            torch.distributed.all_gather_into_tensor(g, lse, group=self.pg)
            mx = g[:, 0].max(dim=0).values
            acc = torch.zeros_like(mx)
            for r in range(self.tp):
                acc += torch.exp(g[r, 0] - mx)
            lse = torch.stack([mx + torch.log(acc), g[:, 1].max(dim=0).values])
        return lse[1] - lse[0]

    def _prefill(self, tokens, start=0, chunk=2048, score=None):
        """prefill(); score: a dict that receives the log-probabilities of score() under "out"."""
        if self.ragged:
            return self._prefill_ragged(tokens, start, chunk, score)
        s, B = self.shape, self.batch
        tokens = torch.as_tensor(tokens, device=self.device)
        if tokens.dim() == 1 and B == 1:
            tokens = tokens.view(1, -1)
        if tokens.dim() != 2 or tokens.shape[0] != B:
            raise ValueError(f"tokens must be [batch={B}, T] (or [T] when batch is 1), got {tuple(tokens.shape)}")
        T = int(tokens.shape[1])
        if T < 1 or start < 0 or start + T > self.cache_len:
            raise ValueError(f"prompt positions [{start}, {start + T}) must lie in the cache [0, {self.cache_len})")
        chunk = min(int(chunk), 65535 // B)
        if chunk < 1:
            raise ValueError("chunk must be >= 1")
        tokens = tokens.to(torch.long)
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        h_last = d_last = None
        if score is not None:
            score["out"] = torch.empty(B, T - 1, dtype=torch.float32, device=self.device)
            nxt = torch.cat([tokens[:, 1:], torch.full((B, 1), -1, dtype=torch.long, device=self.device)], dim=1)  # row t's target
        with torch.no_grad():
            for c0 in range(0, T, chunk):
                n = min(chunk, T - c0)
                h, delta = (self._prefill_chunk_fused if self.fused else self._prefill_chunk_ref)(tokens[:, c0:c0 + n], start + c0, hd, hq, hkv)
                if score is not None and min(n, T - 1 - c0) > 0:
                    lp = self._score_rows(h, delta, nxt[:, c0:c0 + n].reshape(-1)).view(B, n)
                    score["out"][:, c0:c0 + n] = lp[:, :min(n, T - 1 - c0)]
                if c0 + n == T:
                    h_last, d_last = h.view(B, n, s.hidden)[:, -1].contiguous(), delta.view(B, n, s.hidden)[:, -1].contiguous()
            if self.position_keys and start == 0:  # every slot starts a new sequence
                self.seq.add_(1)
            tok = self._prefill_head(h_last, d_last, key_pos=[start + T - 1] * B)
        self.tok.copy_(tok)
        self.pos.fill_((start + T) % self.cache_len)
        return self.tok.clone()

    def _prefill_ragged(self, prompts, start=0, chunk=2048, score=None) -> torch.Tensor:
        """Prefill of a ragged batch: `prompts` holds `batch` entries, each a 1-D token tensor or None (that slot's pos, tok and
        caches stay as they are); a [batch, T] tensor stands for the equal-length list.  `start` is an int or one per slot.  Slot b
        takes in its prompt at positions start_b .. start_b + T_b - 1.  Each chunk takes up to `chunk` tokens from every slot that
        has tokens left (at most 65535 rows in all) and runs them packed in slot order through every block: the linears at
        M = sum of the slots' rows, the _varlen RoPE / append and attention kernels.  With kv_bits 8 the staging rows [0, pos0) are
        dequantised for the slots in the chunk only.  Each slot's last position goes through the final norm, the lm_head and the
        pick (with do_sample: Philox row index = the slot, the counter advancing by one per call; with position keys the slots
        whose prompt starts at position 0 first add one to their seq).  Afterwards pos[b] =
        (start_b + T_b) mod cache_len and tok[b] holds the next token for every prefilled slot; tok is returned and last_logits holds
        the prefilled slots' rows in slot order.  Refilling one slot -- continuous batching -- is a prefill with None for every other
        slot: rows past the slot's new position are never read, so its old cache needs no clearing.
        fused=False: each slot runs the lock-step reference walk (_prefill_chunk_ref) on its own cache."""
        s, B, L = self.shape, self.batch, self.cache_len
        if torch.is_tensor(prompts) and prompts.dim() == 2 and prompts.shape[0] == B:
            prompts = list(prompts.unbind(0))
        if not isinstance(prompts, (list, tuple)) or len(prompts) != B:
            raise ValueError(f"prompts must be a list of batch={B} entries (1-D token tensors or None) or a [batch, T] tensor")
        toks = []
        for b, p in enumerate(prompts):
            if p is None:
                toks.append(None)
                continue
            t = torch.as_tensor(p, device=self.device)
            if t.dim() != 1 or t.numel() < 1:
                raise ValueError(f"prompt {b} must be a non-empty 1-D token tensor, got shape {tuple(t.shape)}")
            toks.append(t.to(torch.long))
        slots = [b for b in range(B) if toks[b] is not None]
        if not slots:
            raise ValueError("prefill needs at least one prompt")
        starts = [start] * B if isinstance(start, int) else list(start)
        if len(starts) != B:
            raise ValueError(f"start must be an int or a list of batch={B} ints")
        for b in slots:
            T = int(toks[b].numel())
            if not (isinstance(starts[b], int) and starts[b] >= 0 and starts[b] + T <= L):
                raise ValueError(f"prompt {b}: positions [{starts[b]}, {starts[b] + T}) must lie in the cache [0, {L})")
        chunk = min(int(chunk), 65535)
        if chunk < 1:
            raise ValueError("chunk must be >= 1")
        if self.kv_pages is not None:  # back every row the prompts write (fresh pages, copy-on-write of a shared partial page)
            self._apply_pages(self.pages.prefill({b: (starts[b], int(toks[b].numel())) for b in slots}))
        if self.spec_k is not None:  # the prompt joins the prompt-lookup history
            for b in slots:
                self.hist[b, starts[b]:starts[b] + toks[b].numel()] = toks[b].to(torch.int32)
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        last = {}
        if score is not None:  # slot b's rows t0 .. t0 + n - 1 score entries t0 .. (the last position has no target)
            out = score["out"] = [None if t is None else torch.empty(t.numel() - 1, dtype=torch.float32, device=self.device) for t in toks]
            nxt = [None if t is None else torch.cat([t[1:], t.new_full((1,), -1)]) for t in toks]

            def scored(h, delta, segs):  # segs: (slot, t0, n) in row order
                lp = self._score_rows(h, delta, torch.cat([nxt[b][t0:t0 + n] for b, t0, n in segs]))
                r = 0
                for b, t0, n in segs:
                    k = max(0, min(n, out[b].numel() - t0))
                    out[b][t0:t0 + k] = lp[r:r + k]
                    r += n
        with torch.no_grad():
            if not self.fused:
                for b in slots:
                    T = int(toks[b].numel())
                    for c0 in range(0, T, chunk):
                        n = min(chunk, T - c0)
                        h, delta = self._prefill_chunk_ref(toks[b][c0:c0 + n].view(1, n), starts[b] + c0, hd, hq, hkv, slot=b)
                        if score is not None:
                            scored(h, delta, [(b, c0, n)])
                    last[b] = (h[-1], delta[-1])
            else:
                done = [0] * B
                while any(toks[b] is not None and done[b] < toks[b].numel() for b in range(B)):
                    budget, n_tok, pos0 = 65535, [0] * B, [0] * B
                    for b in slots:
                        n_tok[b] = min(chunk, int(toks[b].numel()) - done[b], budget)
                        pos0[b] = starts[b] + done[b] if n_tok[b] else 0
                        budget -= n_tok[b]
                    ids = torch.cat([toks[b][done[b]:done[b] + n_tok[b]] for b in slots if n_tok[b]])
                    h, delta = self._prefill_chunk_fused(ids.view(1, -1), 0, hd, hq, hkv, varlen=(pos0, n_tok))
                    if score is not None:
                        scored(h, delta, [(b, done[b], n_tok[b]) for b in slots if n_tok[b]])
                    r = 0
                    for b in range(B):
                        r += n_tok[b]
                        if n_tok[b]:
                            done[b] += n_tok[b]
                            if done[b] == toks[b].numel():
                                last[b] = (h[r - 1], delta[r - 1])
            if self.position_keys and any(starts[b] == 0 for b in slots):  # those slots start new sequences
                new = torch.tensor([b for b in slots if starts[b] == 0], device=self.device)
                self.seq.index_add_(0, new, torch.ones_like(new))
            key_pos = [starts[b] + int(toks[b].numel()) - 1 if toks[b] is not None else 0 for b in range(B)]
            tok = self._prefill_head(torch.stack([last[b][0] for b in slots]), torch.stack([last[b][1] for b in slots]), slots=slots, key_pos=key_pos)
        idx = torch.tensor(slots, device=self.device)
        self.tok.index_copy_(0, idx, tok)
        self.pos.index_copy_(0, idx, torch.tensor([(starts[b] + int(toks[b].numel())) % L for b in slots], device=self.device))
        return self.tok.clone()

    def _prefill_chunk_fused(self, ids, p0, hd, hq, hkv, varlen=None, attn=None):
        """One chunk on the package's kernels; returns the residual stream h [M, hidden] before the last block's MLP delta, and
        that delta (the final norm adds them for the rows it needs).  varlen = (pos0, n_tok) host lists of the ragged batch's slots:
        ids [1, M] packed in slot order and the _varlen kernels (p0 unused).  attn(blk, q, k, v, q_rot, out): the cache append and
        attention step in place of the prefill kernels (the speculative verify pass)."""
        from ._lib import DTYPE_CODE, check, load, ptr, stream_ptr
        lib, s = load(), self.shape
        st = stream_ptr(self.device)
        code = DTYPE_CODE[self.dtype]
        B, n = ids.shape
        M = B * n
        import ctypes
        if varlen is not None:
            B = self.batch
            vp0, vnt = (ctypes.c_int * B)(*varlen[0]), (ctypes.c_int * B)(*varlen[1])
        elif self.kv_bits == 4:  # the lock-step chunk as slots for the 4-bit staging refill
            vp0, vnt = (ctypes.c_int * B)(*[p0] * B), (ctypes.c_int * B)(*[n] * B)
        e = lambda w: torch.empty(M, w, device=self.device, dtype=self.dtype)
        h = self.embed.index_select(0, ids.reshape(-1))  # [M, hidden], row b * n + t
        x, q, k, v, qr, a, o = e(s.hidden), e(hq * hd), e(hkv * hd), e(hkv * hd), e(hq * hd), e(hq * hd), e(s.hidden)
        inter = s.inter // self.tp
        gate, up, act, down = e(inter), e(inter), e(inter), e(s.hidden)
        norm = lambda d, w: check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(h), ptr(d), ptr(w), ptr(x), M, s.hidden, s.rms_eps, code, st))
        delta = None
        kv8 = self._kvq  # 8 or 4 bits: the staging pair, as below
        kvq = f"kv{self.kv_bits}"
        paged = self.kv_pages is not None
        if paged:
            pt, npg = ptr(self.page_table), self.kv_pages
        if kv8 and attn is None and self._kv8_stage is None:  # one staging pair for all layers: [batch, n_kv, cache_len, 128] each
            self._kv8_stage = tuple(torch.zeros(B, hkv, self.cache_len, hd, device=self.device, dtype=self.dtype) for _ in range(2))
        for blk in self.blocks:
            norm(delta, blk["norm1"])
            self._lin(x, (blk["q"], blk["k"], blk["v"]), [q, k, v])
            if attn is not None:
                attn(blk, q, k, v, qr, a)
            elif kv8:
                # staging rows [0, p0) dequantised from the 8-bit cache, rows [p0, p0 + n) written by the rows kernel; the attention
                # kernel is the one of the fp16 cache, reading the staging pair
                kst, vst = self._kv8_stage
                for bi in range(0 if paged or self.kv_bits == 4 else B):
                    sp0 = p0 if varlen is None else (varlen[0][bi] if varlen[1][bi] else 0)  # slots outside the chunk: nothing
                    for hh in range(hkv):
                        for c, dst in (("k", kst), ("v", vst)):
                            if sp0 > 0:
                                check(lib.hqq_b200_dequantize(ptr(blk[c + "_cache"][bi, hh]), ptr(blk[c + "_scale"][bi, hh]), ptr(blk[c + "_zero"][bi, hh]),
                                                              ptr(dst[bi, hh]), sp0, hd, self.kv_group_size, 8, 1, code, st))
                if self.kv_bits == 4 and not paged:  # every row is packed on its own: one launch refills the staging rows [0, pos0)
                    check(lib.hqq_b200_glue_kv4_stage(ptr(blk["k_cache"]), ptr(blk["k_scale"]), ptr(blk["k_zero"]), ptr(blk["v_cache"]), ptr(blk["v_scale"]),
                                                      ptr(blk["v_zero"]), ptr(kst), ptr(vst), vp0, vnt, hkv, self.cache_len, hd, self.kv_group_size, B,
                                                      code, st))
                if paged:  # one launch refills the staging rows [0, pos0) of the slots in the chunk, through the table
                    check(getattr(lib, f"hqq_b200_glue_{kvq}_stage_paged")(ptr(blk["k_cache"]), ptr(blk["k_scale"]), ptr(blk["k_zero"]), ptr(blk["v_cache"]),
                                                            ptr(blk["v_scale"]), ptr(blk["v_zero"]), pt, ptr(kst), ptr(vst), vp0, vnt, hkv, self.cache_len, hd,
                                                            self.kv_group_size, B, npg, code, st))
                    check(getattr(lib, f"hqq_b200_glue_rope_append_rows_{kvq}_paged")(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                                       ptr(blk["k_scale"]), ptr(blk["k_zero"]), ptr(blk["v_cache"]), ptr(blk["v_scale"]),
                                                                       ptr(blk["v_zero"]), pt, ptr(kst), ptr(vst), ptr(qr), vp0, vnt, hq, hkv, self.cache_len,
                                                                       hd, self.kv_group_size, B, npg, code, st))
                elif varlen is not None:
                    check(getattr(lib, f"hqq_b200_glue_rope_append_rows_{kvq}_varlen")(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                                        ptr(blk["k_scale"]), ptr(blk["k_zero"]), ptr(blk["v_cache"]), ptr(blk["v_scale"]),
                                                                        ptr(blk["v_zero"]), ptr(kst), ptr(vst), ptr(qr), vp0, vnt, hq, hkv, self.cache_len, hd,
                                                                        self.kv_group_size, B, code, st))
                else:
                    check(getattr(lib, f"hqq_b200_glue_rope_append_rows_{kvq}")(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]), ptr(blk["k_scale"]),
                                                                 ptr(blk["k_zero"]), ptr(blk["v_cache"]), ptr(blk["v_scale"]), ptr(blk["v_zero"]), ptr(kst),
                                                                 ptr(vst), ptr(qr), p0, n, hq, hkv, self.cache_len, hd, self.kv_group_size, B, code, st))
                kc, vc = kst, vst
            elif paged:
                check(lib.hqq_b200_glue_rope_append_rows_paged(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]), ptr(blk["v_cache"]),
                                                               pt, ptr(qr), vp0, vnt, hq, hkv, self.cache_len, hd, B, npg, code, st))
                kc, vc = blk["k_cache"], blk["v_cache"]
            elif varlen is not None:
                check(lib.hqq_b200_glue_rope_append_rows_varlen(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                                ptr(blk["v_cache"]), ptr(qr), vp0, vnt, hq, hkv, self.cache_len, hd, B, code, st))
                kc, vc = blk["k_cache"], blk["v_cache"]
            else:
                check(lib.hqq_b200_glue_rope_append_rows(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]), ptr(blk["v_cache"]),
                                                         ptr(qr), p0, n, hq, hkv, self.cache_len, hd, B, code, st))
                kc, vc = blk["k_cache"], blk["v_cache"]
            if attn is not None:
                pass  # the hook's attention output is in a already
            elif paged and not kv8:
                check(lib.hqq_b200_glue_attn_prefill_paged(ptr(qr), ptr(kc), ptr(vc), pt, ptr(a), vp0, vnt, hq, hkv, self.cache_len, hd, B, npg, code, st))
            elif varlen is not None:
                check(lib.hqq_b200_glue_attn_prefill_varlen(ptr(qr), ptr(kc), ptr(vc), ptr(a), vp0, vnt, hq, hkv, self.cache_len, hd, B, code, st))
            else:
                check(lib.hqq_b200_glue_attn_prefill(ptr(qr), ptr(kc), ptr(vc), ptr(a), p0, n, hq, hkv, self.cache_len, hd, B, code, st))
            self._lin(a, (blk["o"],), [o])
            if self.tp > 1:
                torch.distributed.all_reduce(o, group=self.pg)
            norm(o, blk["norm2"])
            self._lin(x, (blk["gate"], blk["up"]), [gate, up])
            check(lib.hqq_b200_glue_silu_mul(ptr(gate), ptr(up), ptr(act), M * inter, code, st))
            self._lin(act, (blk["down"],), [down])
            if self.tp > 1:
                torch.distributed.all_reduce(down, group=self.pg)
            delta = down
        return h, delta

    def _prefill_chunk_ref(self, ids, p0, hd, hq, hkv, slot=None):
        """The same chunk on framework ops (fused=False); slot: ids [1, n] of that slot only, on that slot's caches (kv_pages: gathered
        through the table, and the chunk's rows stored back through it)."""
        s = self.shape
        B, n = ids.shape
        M = B * n
        h = self.embed.index_select(0, ids.reshape(-1))
        cos, sin = self.cos[p0:p0 + n].view(1, n, 1, hd), self.sin[p0:p0 + n].view(1, n, 1, hd)
        end = p0 + n
        mask = torch.arange(end, device=self.device).view(1, end) <= torch.arange(p0, end, device=self.device).view(n, 1)  # [n, end]
        delta = None
        for blk in self.blocks:
            if slot is None:
                cb = blk
            elif self.kv_pages is None:
                cb = {n: t[slot:slot + 1] for n, t in blk.items() if n.startswith(("k_", "v_"))}
            else:
                cb = {n: t[slot:slot + 1].clone() for n, t in self.cache_view(blk).items()}
            if delta is not None:
                h = h + delta
            x = F.rms_norm(h, (s.hidden,), blk["norm1"], s.rms_eps)
            q, k, v = self._multi(x, (blk["q"], blk["k"], blk["v"]))
            q = self._rope(q.view(B, n, hq, hd), cos, sin)
            k = self._rope(k.view(B, n, hkv, hd), cos, sin)
            if self._kvq:
                self._kv8_write(cb, k.transpose(1, 2), v.view(B, n, hkv, hd).transpose(1, 2), torch.arange(p0, end, device=self.device))
                kc, vc = self._kv8_read(cb, end)
            else:
                cb["k_cache"][:, :, p0:end] = k.transpose(1, 2)
                cb["v_cache"][:, :, p0:end] = v.view(B, n, hkv, hd).transpose(1, 2)
                kc, vc = cb["k_cache"][:, :, :end], cb["v_cache"][:, :, :end]
            if slot is not None and self.kv_pages is not None:  # the chunk's rows into their pages
                rows = torch.arange(p0, end, device=self.device)
                at = (self.page_table[slot, rows // KV_PAGE].long(), slice(None), rows % KV_PAGE)
                for name, t in cb.items():
                    blk[name][at] = t[0, :, p0:end].transpose(0, 1)
            a = F.scaled_dot_product_attention(q.transpose(1, 2), kc, vc, attn_mask=mask, enable_gqa=True)
            o = blk["o"](a.transpose(1, 2).reshape(M, hq * hd))
            if self.tp > 1:
                torch.distributed.all_reduce(o, group=self.pg)
            h = h + o
            x = F.rms_norm(h, (s.hidden,), blk["norm2"], s.rms_eps)
            g, u = self._multi(x, (blk["gate"], blk["up"]))
            delta = blk["down"](F.silu(g) * u)
            if self.tp > 1:
                torch.distributed.all_reduce(delta, group=self.pg)
        return h, delta

    def _prefill_head(self, h, delta, slots=None, key_pos=None):
        """Final norm, lm_head and greedy pick for the last position of each sequence: h, delta [batch, hidden].  slots (ragged): h,
        delta hold the rows of those slots; with do_sample row b is drawn with Philox row index b, its slot.  key_pos: host list of
        every slot's last prompt position, the position keys' p (slots outside a ragged subset: any value, their draws discarded)."""
        s, B = self.shape, h.shape[0]
        kp = torch.tensor(key_pos, dtype=torch.long, device=self.device) if self.position_keys else None

        def full(lg):  # do_sample on a ragged subset: the rows at their slots in a [batch, vocab / tp] block (the others discarded)
            if slots is None:
                return lg
            f = torch.zeros(self.batch, lg.shape[1], dtype=lg.dtype, device=lg.device)
            f[torch.tensor(slots, device=lg.device)] = lg
            return f

        pick = (lambda t: t) if slots is None else (lambda t: t[torch.tensor(slots, device=t.device)])
        if not self.fused:
            x = F.rms_norm(h + delta, (s.hidden,), self.final_norm, s.rms_eps)
            logits = torch.matmul(x, self.lm_head.t())
            self.last_logits = logits
            if self.do_sample:
                tok = pick(self._sample_ref(full(logits), kp))
                self._sample_ctr.add_(1)
                return tok
            if self.tp == 1:
                return torch.argmax(logits, dim=-1)
            val, idx = torch.max(logits.float(), dim=-1)
            gmax = val.clone()
            torch.distributed.all_reduce(gmax, op=torch.distributed.ReduceOp.MAX, group=self.pg)
            cand = torch.where(val == gmax, idx + self.rank * self.vocab_shard, torch.full_like(idx, s.vocab))
            torch.distributed.all_reduce(cand, op=torch.distributed.ReduceOp.MIN, group=self.pg)
            return cand
        from ._lib import DTYPE_CODE, check, load, ptr, stream_ptr
        lib = load()
        st = stream_ptr(self.device)
        code = DTYPE_CODE[self.dtype]
        x = torch.empty_like(h)
        check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(h), ptr(delta), ptr(self.final_norm), ptr(x), B, s.hidden, s.rms_eps, code, st))
        self.last_logits = torch.matmul(x, self.lm_head.t())
        if self.do_sample:
            rows = full(self.last_logits)
            tok = torch.empty(rows.shape[0], dtype=torch.long, device=self.device)
            self._sample(lib, self._sample_rows(rows, self._sample_buffers(rows.shape[0])), tok, code, st, pos=kp)
            self._sample_ctr.add_(1)
            return pick(tok)
        # the argmax kernel reads 16-byte vectors: every row starts on a 16-byte boundary whatever the vocabulary shard's length
        n = self.vocab_shard
        rows = torch.empty(B, -(-n // 8) * 8, dtype=self.dtype, device=self.device)
        rows[:, :n].copy_(self.last_logits)
        key = torch.empty(B, dtype=torch.long, device=self.device)
        for b in range(B):  # {value : 0xFFFFFFFF - global index} keys: their MAX over the vocabulary shards is the first global argmax
            check(lib.hqq_b200_glue_argmax_key(ptr(rows[b]), n, self.rank * n, ptr(key[b:]), code, st))
        if self.tp > 1:
            torch.distributed.all_reduce(key, op=torch.distributed.ReduceOp.MAX, group=self.pg)
        return 0xFFFFFFFF - torch.bitwise_and(key, 0xFFFFFFFF)

    def _alloc_bufs(self):
        s, dev, dt = self.shape, self.device, self.dtype
        z = lambda n: torch.zeros(self.batch, n, device=dev, dtype=dt)
        tp = self.tp
        self._bufs = {"h": z(s.hidden), "h2": z(s.hidden), "x": z(s.hidden), "q": z(s.n_heads // tp * s.head_dim), "k": z(s.n_kv_heads // tp * s.head_dim),
                      "v": z(s.n_kv_heads // tp * s.head_dim), "a": z(s.n_heads // tp * s.head_dim), "o": z(s.hidden),
                      "gate": z(s.inter // tp), "up": z(s.inter // tp), "act": z(s.inter // tp), "down": z(s.hidden), "logits": z(self.vocab_shard),
                      "key": torch.zeros(1, dtype=torch.long, device=dev)}
        if self.do_sample:
            self._bufs.update(self._sample_buffers(self.batch))
            if self.position_keys and self.pos.numel() != self.batch:
                self._bufs["sample_pos"] = torch.zeros(self.batch, dtype=torch.long, device=dev)
        if self.attn_kernel != "single":  # partials + tickets, zeroed once: every launch leaves the tickets at zero
            from ._lib import load
            with torch.cuda.device(dev):
                nbytes = load().hqq_b200_glue_rope_attn_decode_split_workspace_bytes(s.n_heads // tp, s.n_kv_heads // tp, s.head_dim, self.batch)
            self._bufs["attn_ws"] = torch.zeros(nbytes, dtype=torch.uint8, device=dev)

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
        if self.kv_pages is not None:
            self.pages.pos = [0] * self.batch
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            step()
        return self.graph

    def reset_state(self, token: int = 1):
        """Position 0, empty KV caches, `token` as the first input: the state every token-stream comparison starts from."""
        self.tok.fill_(token)
        self.pos.zero_()
        self._sample_ctr.zero_()
        if self.seq is not None:
            self.seq.zero_()
        if self.kv_pages is not None:  # every page free, every entry the sink, every slot active at position 0
            self.pages.reset()
            self.page_table.fill_(self.kv_pages)
        if self.spec_k is not None:
            self.hist.zero_()
        for blk in self.blocks:
            for name in ("k_cache", "v_cache", "k_scale", "k_zero", "v_scale", "v_zero"):
                if name in blk:
                    blk[name].zero_()
        if hasattr(self, "_bufs"):
            for t in self._bufs.values():
                t.zero_()

    def decode(self, feed_back: bool = True):
        """Replay one step; with feed_back the produced token becomes the next input (device-side copy).  With kv_pages, callers
        must step through decode(), not a bare graph.replay(): before the replay a slot about to enter a page gets it here (stream-
        ordered table writes, no sync).  A bare replay cannot address outside the pools, but its writes at a page edge go to the sink."""
        if self.kv_pages is not None:
            self._apply_pages(self.pages.step())
        self.graph.replay()
        if feed_back:
            self.tok.copy_(self.next_tok)

    # ---- speculative decoding (spec_k)
    def _spec_window_ids(self):
        """The verify rows [batch, K + 1]: tok, then the drafts (a -1 sentinel embeds as token 0: it never matches, so no row
        after it is accepted)."""
        return torch.cat([self.tok.view(-1, 1), self._spec_drafts.clamp_min(0)], dim=1)

    def _greedy(self, logits):
        """Targets of logits rows [M, vocab / tp], first index on ties: torch.argmax at tp = 1, else the global maximum and then
        the lowest global index that attains it (two small all-reduces), as the batched head does."""
        if self.tp == 1:
            return torch.argmax(logits, dim=-1)
        val, idx = torch.max(logits.float(), dim=-1)
        gmax = val.clone()
        torch.distributed.all_reduce(gmax, op=torch.distributed.ReduceOp.MAX, group=self.pg)
        cand = torch.where(val == gmax, idx + self.rank * self.vocab_shard, torch.full_like(idx, self.shape.vocab))
        torch.distributed.all_reduce(cand, op=torch.distributed.ReduceOp.MIN, group=self.pg)
        return cand

    def verify_fused(self):
        """One speculative verify step on the package's kernels: the window [tok, d1 .. dK] of every slot runs the prefill block walk
        (_prefill_chunk_fused) at M = batch (K + 1) rows, with the device-position append and the verify attention as its attention
        step; every row goes through the final norm and the lm_head, the targets are the rows' greedy picks (do_sample: one
        hqq_b200_glue_sample_pos launch over all rows, after one all-gather under tensor parallelism), and one
        hqq_b200_glue_spec_accept launch emits the accepted tokens and advances pos, tok, next_tok and hist on the device."""
        from ._lib import DTYPE_CODE, check, load, ptr, stream_ptr
        lib, s = load(), self.shape
        st = stream_ptr(self.device)
        code = DTYPE_CODE[self.dtype]
        B, K, L = self.batch, self.spec_k, self.cache_len
        T = K + 1
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        ws = self._bufs["verify_ws"]

        def attn(blk, q, k, v, qr, a):
            if self._kvq:
                c8 = [ptr(blk[n]) for n in ("k_cache", "k_scale", "k_zero", "v_cache", "v_scale", "v_zero")]
                gs = self.kv_group_size
                kvq = f"kv{self.kv_bits}"
                if self.kv_pages is None:
                    check(getattr(lib, f"hqq_b200_glue_rope_append_rows_{kvq}_devpos")(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), *c8, ptr(qr), ptr(self.pos), T,
                                                                        hq, hkv, L, hd, gs, B, code, st))
                    check(getattr(lib, f"hqq_b200_glue_attn_verify_split_{kvq}")(ptr(qr), *c8, ptr(self.pos), ptr(a), ptr(ws), hq, hkv, L, hd, gs, T, B, code, st))
                    return
                pt = ptr(self.page_table)
                check(getattr(lib, f"hqq_b200_glue_rope_append_rows_{kvq}_devpos_paged")(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), *c8, pt, ptr(qr),
                                                                          ptr(self.pos), T, hq, hkv, L, hd, gs, B, self.kv_pages, code, st))
                check(getattr(lib, f"hqq_b200_glue_attn_verify_split_{kvq}_paged")(ptr(qr), *c8, pt, ptr(self.pos), ptr(a), ptr(ws), hq, hkv, L, hd, gs, T, B,
                                                                    self.kv_pages, code, st))
                return
            if self.kv_pages is None:
                check(lib.hqq_b200_glue_rope_append_rows_devpos(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                                ptr(blk["v_cache"]), ptr(qr), ptr(self.pos), T, hq, hkv, L, hd, B, code, st))
                check(lib.hqq_b200_glue_attn_verify_split(ptr(qr), ptr(blk["k_cache"]), ptr(blk["v_cache"]), ptr(self.pos), ptr(a), ptr(ws), hq, hkv, L,
                                                          hd, T, B, code, st))
                return
            pt = ptr(self.page_table)
            check(lib.hqq_b200_glue_rope_append_rows_devpos_paged(ptr(q), ptr(k), ptr(v), ptr(self.cos), ptr(self.sin), ptr(blk["k_cache"]),
                                                                  ptr(blk["v_cache"]), pt, ptr(qr), ptr(self.pos), T, hq, hkv, L, hd, B, self.kv_pages,
                                                                  code, st))
            check(lib.hqq_b200_glue_attn_verify_split_paged(ptr(qr), ptr(blk["k_cache"]), ptr(blk["v_cache"]), pt, ptr(self.pos), ptr(a), ptr(ws), hq,
                                                            hkv, L, hd, T, B, self.kv_pages, code, st))

        h, delta = self._prefill_chunk_fused(self._spec_window_ids(), 0, hd, hq, hkv, attn=attn)
        x = torch.empty_like(h)
        check(lib.hqq_b200_glue_add_rmsnorm_rows(ptr(h), ptr(delta), ptr(self.final_norm), ptr(x), B * T, s.hidden, s.rms_eps, code, st))
        logits = self._bufs["verify_logits"]
        torch.matmul(x, self.lm_head.t(), out=logits)
        if self.do_sample:  # position keys: row b T + t is drawn at position pos[b] + t
            self._sample(lib, self._sample_rows(logits, self._verify_sample_bufs), self._spec_targets, code, st, pos=self.pos, T=T)
        else:
            self._spec_targets.copy_(self._greedy(logits))
        check(lib.hqq_b200_glue_spec_accept(ptr(self._spec_targets), ptr(self._spec_drafts), ptr(self.pos), ptr(self.tok), ptr(self.next_tok),
                                            ptr(self.hist), ptr(self._spec_tokens), ptr(self._spec_n_new), L, K, B, st))

    def verify(self):
        """The same verify step on framework ops (fused=False), the reference: per-row RoPE, the window's valid rows (t < n[b]) written
        into the caches (through the page table when paged; kv_bits 8: quantised by kv8_quantize_rows, attention over the
        dequantised cache), SDPA with the per-slot causal masks key <= pos[b] + t, the head, the targets (do_sample: sample_tokens
        with the position keys of each row), and the accept rule restated with tensor ops."""
        s, B, K, L = self.shape, self.batch, self.spec_k, self.cache_len
        T = K + 1
        hd, hq, hkv = s.head_dim, s.n_heads // self.tp, s.n_kv_heads // self.tp
        dev = self.device
        ids = self._spec_window_ids()
        rows = self.pos.view(B, 1) + torch.arange(T, device=dev).view(1, T)  # [B, T] positions
        n = torch.clamp(L - self.pos, max=T)
        valid = torch.arange(T, device=dev).view(1, T) < n.view(B, 1)
        at_rows = torch.where(valid, rows, torch.zeros_like(rows))  # rows past the cache: any RoPE row, never written
        cos, sin = self.cos[at_rows].view(B, T, 1, hd), self.sin[at_rows].view(B, T, 1, hd)
        mask = (self.arange.view(1, 1, L) <= rows.view(B, T, 1)).view(B, 1, T, L)
        bi, ti = valid.nonzero(as_tuple=True)
        p = rows[bi, ti]
        at = (bi, slice(None), p) if self.kv_pages is None else (self.page_table[bi, p // KV_PAGE].long(), slice(None), p % KV_PAGE)
        h = self.embed.index_select(0, ids.reshape(-1))
        for blk in self.blocks:
            x = F.rms_norm(h, (s.hidden,), blk["norm1"], s.rms_eps)
            q, k, v = self._multi(x, (blk["q"], blk["k"], blk["v"]))
            q = self._rope(q.view(B, T, hq, hd), cos, sin)
            k = self._rope(k.view(B, T, hkv, hd), cos, sin)
            for name, x in (("k", k[bi, ti]), ("v", v.view(B, T, hkv, hd)[bi, ti])):
                if self._kvq:
                    for suffix, val in zip(("_cache", "_scale", "_zero"), kv8_quantize_rows(x, self.kv_group_size, self.kv_bits)):
                        blk[name + suffix][at] = val
                else:
                    blk[name + "_cache"][at] = x
            cv = self.cache_view(blk)
            kc, vc = self._kv8_read(cv, L) if self._kvq else (cv["k_cache"], cv["v_cache"])
            a = F.scaled_dot_product_attention(q.transpose(1, 2), kc, vc, attn_mask=mask, enable_gqa=True)
            o = blk["o"](a.transpose(1, 2).reshape(B * T, hq * hd))
            if self.tp > 1:
                torch.distributed.all_reduce(o, group=self.pg)
            h = h + o
            x = F.rms_norm(h, (s.hidden,), blk["norm2"], s.rms_eps)
            g, u = self._multi(x, (blk["gate"], blk["up"]))
            y = blk["down"](F.silu(g) * u)
            if self.tp > 1:
                torch.distributed.all_reduce(y, group=self.pg)
            h = h + y
        h = F.rms_norm(h, (s.hidden,), self.final_norm, s.rms_eps)
        logits = torch.matmul(h, self.lm_head.t())
        self.spec_logits = logits.view(B, T, -1)
        if self.do_sample:  # position keys: row t of slot b at position pos[b] + t
            tg = torch.stack([self._sample_ref(self.spec_logits[:, t], self.pos + t) for t in range(T)], dim=1)
        else:
            tg = self._greedy(logits).view(B, T)
        d = self._spec_drafts
        ok = (d == tg[:, :K]) & (torch.arange(1, T, device=dev).view(1, K) < n.view(B, 1))
        a = torch.cumprod(ok.long(), dim=1).sum(dim=1)  # accepted drafts
        i = torch.arange(T, device=dev).view(1, T)
        t_a = tg.gather(1, a.view(B, 1))
        self._spec_tokens.copy_(torch.where(i < a.view(B, 1), torch.cat([d, d[:, :1]], 1), torch.where(i == a.view(B, 1), t_a, -1)))
        window = torch.cat([self.tok.view(B, 1), d], 1)
        for r in range(T):  # hist[pos + r] = window[r] for r <= a
            idx = (self.pos + r).clamp(max=L - 1).view(B, 1)
            cur = self.hist.gather(1, idx)
            self.hist.scatter_(1, idx, torch.where((r <= a).view(B, 1), window[:, r:r + 1].to(torch.int32), cur))
        self._spec_targets.copy_(tg.view(-1))
        self._spec_n_new.copy_(a + 1)
        self.pos.copy_((self.pos + a + 1) % L)
        self.tok.copy_(t_a.view(B))
        self.next_tok.copy_(t_a.view(B))

    def capture_spec(self, warmup: int = 3):
        """Capture one verify step (verify_fused) into self.spec_graph.  The warm-up runs on the current state and puts back pos,
        tok, next_tok and hist afterwards; the cache rows it wrote lie past the slots' positions, where no step reads.  fused=False
        needs no capture: decode_spec() runs verify() eagerly."""
        if self.spec_k is None:
            raise ValueError("capture_spec needs spec_k")
        if not self.fused:
            raise ValueError("capture_spec needs a fused model (fused=False runs verify() eagerly in decode_spec)")
        if not hasattr(self, "_bufs"):
            self._alloc_bufs()
        if "verify_ws" not in self._bufs:
            from ._lib import load
            s, tp, T = self.shape, self.tp, self.spec_k + 1
            with torch.cuda.device(self.device):
                nbytes = load().hqq_b200_glue_attn_verify_split_workspace_bytes(s.n_heads // tp, s.n_kv_heads // tp, s.head_dim, T, self.batch)
            self._bufs["verify_ws"] = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
            self._bufs["verify_logits"] = torch.zeros(self.batch * T, self.vocab_shard, dtype=self.dtype, device=self.device)
            if self.do_sample:
                self._verify_sample_bufs = self._sample_buffers(self.batch * T)
        self.spec_logits = self._bufs["verify_logits"].view(self.batch, self.spec_k + 1, -1)
        saved = [t.clone() for t in (self.pos, self.tok, self.next_tok, self.hist, self._spec_drafts)]
        self._spec_drafts.fill_(-1)
        st = torch.cuda.Stream(device=self.device)
        st.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(st), torch.no_grad():
            for _ in range(warmup):
                self.verify_fused()
        torch.cuda.current_stream(self.device).wait_stream(st)
        torch.cuda.synchronize(self.device)
        for t, v in zip((self.pos, self.tok, self.next_tok, self.hist, self._spec_drafts), saved):
            t.copy_(v)
        self.spec_graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.spec_graph):
            self.verify_fused()
        return self.spec_graph

    def decode_spec(self, drafts: torch.Tensor | None = None):
        """One speculative step for every slot: drafts from prompt lookup (hqq_b200_glue_ngram_draft over hist, launched in front of
        the replay) or the caller's device int64 [batch, K] (-1 for none), then the captured verify step (fused=False: verify()).
        Caller drafts outside [0, vocab) count as -1 (mapped on the device).
        Returns (tokens [batch, K + 1] with -1 after the emitted ones, n_new [batch]) as device tensors; tok / next_tok hold the last
        emitted token, so decode() and decode_spec() may be interleaved.  No synchronisation, except with kv_pages: the pages past
        the accepted tokens are returned by spec_advance, which reads n_new to the host once per call."""
        from ._lib import check, load, ptr, stream_ptr
        if self.spec_k is None:
            raise ValueError("decode_spec needs spec_k")
        B, K = self.batch, self.spec_k
        if drafts is None:
            check(load().hqq_b200_glue_ngram_draft(ptr(self.hist), ptr(self.pos), ptr(self.tok), ptr(self._spec_drafts), self.cache_len, K, B,
                                                   stream_ptr(self.device)))
        else:
            if not (torch.is_tensor(drafts) and drafts.shape == (B, K) and drafts.device == self.device and not drafts.is_floating_point()):
                raise ValueError(f"drafts must be an integer tensor [batch={B}, K={K}] on {self.device}")
            self._spec_drafts.copy_(torch.where((drafts >= 0) & (drafts < self.shape.vocab), drafts, -1))
        if self.kv_pages is not None:
            self._apply_pages(self.pages.spec_window(K))
        with torch.no_grad():
            if self.fused:
                if self.spec_graph is None:
                    raise RuntimeError("decode_spec on a fused model needs capture_spec() first")
                self.spec_graph.replay()
            else:
                self.verify()
        if self.kv_pages is not None:
            self._apply_pages(self.pages.spec_advance(self._spec_n_new.tolist()))
        return self._spec_tokens.clone(), self._spec_n_new.clone()


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
